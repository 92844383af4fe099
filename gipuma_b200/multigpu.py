"""Multi-GPU drivers for the PatchMatch hot path: one process per GPU, `torch.distributed` for the plumbing.

Two axes shard (SURVEY.md §8e); the reference itself is single-GPU (main.cpp:658-692).

1. **Reference-view batch** — independent units.  The reference runs one process per reference image
   (scripts/dtu_fast.sh:30-55); `assign_reference_views` deals reference views round-robin to ranks and
   `run_reference_view_batch` runs each on the rank's own context.  No data-path collective; `bench.py --gpus N` is
   this mode (weak scaling).

2. **Source-view shard** inside one reference view (BASELINE config 4: 47 views over 4 GPUs).  Per-view costs are
   independent; only their combination needs all views (gipuma.cu:742-806).  `north_star` words this as "allreduce
   of best cost/plane", which is NOT the reference's rule (best-n over ALL views, summed in ascending order); the
   exact formulation used here: per stage, every rank exports per pixel and hypothesis slot its ascending n_best
   smallest per-view costs, the lists are all-gathered (ncclAllGather over NVLink, issued by gpm_shard_run behind the
   C-ABI), and every rank merges, combines and applies the accept logic redundantly (fused into the next stage).  State
   stays bit-identical on all ranks and identical to a single-GPU run.  Collectives per iteration:
   2 colours x (1 propagation + S refinement steps) = 8 on DTU parameters; payload per rank and colour:
   H*ceil(W/2)*8*n_best*4 B for propagation (7.4 MB at 640x480, n_best 3), 1/8 of that per refinement step.
   The exchange is a genuine step of the algorithm (a hypothesis can only be accepted once all views are known), so
   it cannot be fused away; it is tiny next to the sampling work.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import numpy as np

MAXCOST = 1000.0


# ----------------------------------------------------------------------------------------------------------------
# partitioning (pure host logic)
# ----------------------------------------------------------------------------------------------------------------

def assign_reference_views(n_reference_views: int, rank: int, world: int) -> List[int]:
    """Reference views r, r+world, ... for `rank` (the shell loop of scripts/dtu_fast.sh:30-55, dealt round-robin)."""
    return list(range(rank, n_reference_views, world))


def partition_views(n_views: int, world: int) -> List[List[int]]:
    """Positions 0..n_views-1 of viewSelectionSubset split into `world` contiguous, balanced shards."""
    base, extra = divmod(n_views, world)
    out, start = [], 0
    for r in range(world):
        n = base + (1 if r < extra else 0)
        out.append(list(range(start, start + n)))
        start += n
    return out


def local_topn(costs: np.ndarray, n_best: int) -> np.ndarray:
    """Ascending n_best smallest of the per-view costs along the last axis, padded with +inf; costs >= MAXCOST are
    clamped to MAXCOST first (gipuma.cu:771-774).  NumPy mirror of the device function `local_topn`."""
    c = np.minimum(np.asarray(costs, dtype=np.float32), np.float32(MAXCOST))
    pad = max(0, n_best - c.shape[-1])
    if pad:
        c = np.concatenate([c, np.full(c.shape[:-1] + (pad,), np.inf, np.float32)], axis=-1)
    return np.sort(c, axis=-1)[..., :n_best]


def merge_topn(gathered: np.ndarray, n_best: int) -> np.ndarray:
    """gathered: [world, ..., n_best] ascending lists.  Returns the combined cost exactly as `shard_merge` /
    pmCostMultiview_cu (COMB_BEST_N) do: the n_best smallest valid (< MAXCOST) costs summed in ascending order in
    float32, divided by their count; MAXCOST if none; +inf if no rank has a finite entry (a slot every rank skipped)."""
    g = np.moveaxis(np.asarray(gathered, dtype=np.float32), 0, -2)          # [..., world, n_best]
    flat = np.sort(g.reshape(g.shape[:-2] + (-1,)), axis=-1)[..., :n_best]
    skipped = flat[..., 0] == np.float32(np.inf)
    valid = flat < np.float32(MAXCOST)
    total = np.zeros(flat.shape[:-1], np.float32)
    for i in range(flat.shape[-1]):                                          # ascending, float32, like the device loop
        total = np.where(valid[..., i], (total + np.where(valid[..., i], flat[..., i], 0)).astype(np.float32), total)
    cnt = valid.sum(axis=-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        cost = np.where(cnt > 0, total / np.maximum(cnt, 1).astype(np.float32), np.float32(MAXCOST)).astype(np.float32)
    cost = np.where((cost != cost) | (cost > MAXCOST) | (cost < 0), np.float32(MAXCOST), cost)
    return np.where(skipped, np.float32(np.inf), cost).astype(np.float32)


# ----------------------------------------------------------------------------------------------------------------
# reference-view batch
# ----------------------------------------------------------------------------------------------------------------

def run_reference_view_batch(images, Ps, params, refs: Sequence[int], devices: Sequence[int] = (0,), **kw):
    """The shell loop of scripts/dtu_fast.sh:30-55 in one process: gpm_batch_run (native host C++, gipuma_b200/csrc/gpm_batch.cpp)
    — a worker thread and context per device, ONE page-locked copy of the image set shared by all of them, reference views
    taken from a common queue.  Thin wrapper over api.batch_run; returns (norm4, cost, stats)."""
    from . import api
    return api.batch_run(images, Ps, params, list(refs), devices=list(devices), **kw)


# ----------------------------------------------------------------------------------------------------------------
# both axes at once (BASELINE config 5: "view-shard + ref-view batch")
# ----------------------------------------------------------------------------------------------------------------

def hybrid_layout(world: int, shard: int):
    """Split `world` ranks into world/shard groups of `shard` consecutive ranks: the groups work on different reference
    views (batch axis), the ranks inside a group shard the source views of their group's current reference view.
    Returns (group_of_rank, rank_in_group, members_of_group) lists."""
    if shard < 1 or world % shard:
        raise ValueError("world size must be a multiple of the view-shard width")
    group_of = [r // shard for r in range(world)]
    rank_in = [r % shard for r in range(world)]
    members = [list(range(g * shard, (g + 1) * shard)) for g in range(world // shard)]
    return group_of, rank_in, members


def run_hybrid(make_scene: Callable[[int], object], n_reference_views: int, rank: int, world: int, shard: int,
               device: int = 0, on_result: Optional[Callable] = None, exchange: str = "nccl",
               propagation: str = "fixed", view_selection: str = "off", planar_prior=None) -> List[float]:
    """Reference views are dealt round-robin to world/shard groups; inside a group the source views are sharded and
    combined with one all-gather per stage over the group's own communicator (`exchange` must be "nccl").  `propagation`
    and `view_selection` as ViewShardRunner.  Returns wall seconds per reference view."""
    import time
    import torch
    import torch.distributed as dist
    from . import api
    _check_exchange(exchange)
    api.check_propagation(propagation)
    _check_view_selection(view_selection)
    _check_planar_prior(planar_prior)
    group_of, rank_in, members = hybrid_layout(world, shard)
    groups = [dist.new_group(ranks=m) if world > 1 else None for m in members]     # every rank creates every group
    my_group = group_of[rank]
    times = []
    for ref in assign_reference_views(n_reference_views, my_group, len(members)):
        sc = make_scene(ref)
        runner = ViewShardRunner(sc, rank_in[rank], shard, device=device, group=groups[my_group], exchange=exchange,
                                  propagation=propagation)
        torch.cuda.synchronize(device)
        t0 = time.perf_counter()
        n4, c = runner.run()
        torch.cuda.synchronize(device)
        times.append(time.perf_counter() - t0)
        if on_result is not None and rank_in[rank] == 0:
            on_result(ref, n4, c)
        runner.close()
    return times


# ----------------------------------------------------------------------------------------------------------------
# source-view shard
# ----------------------------------------------------------------------------------------------------------------

def _check_exchange(exchange: str):
    if exchange == "p2p":
        raise ValueError('exchange="p2p": the fused peer-memory exchange was removed (DESIGN.md §8); use exchange="nccl"')
    if exchange != "nccl":
        raise ValueError(f"unknown exchange {exchange!r}: the source-view shard exchanges with NCCL only")


def _check_view_selection(view_selection: str):
    from . import api
    api.view_sel(view_selection)
    if view_selection != "off":
        raise ValueError("view_selection=%r: the source-view shard has no joint view selection (its exchange carries top-n "
                         "lists, not per-view costs)" % (view_selection,))


def _check_planar_prior(planar_prior):
    if planar_prior is not None:
        raise ValueError("planar_prior: the source-view shard has no planar prior (its exchange carries top-n lists of the "
                         "photometric cost)")


class ViewShardRunner:
    """One reference view, source views sharded over `world` ranks.  All device work runs behind the C-ABI
    (gpm_shard_run): one stage kernel + ncclAllGather per exchange stage.  `exchange` must be "nccl"; the attribute of
    the same name is "nccl", or "none" for a single rank.  torch.distributed is only used at set-up, to pass the NCCL
    unique id around.  `propagation` ("fixed" or "adaptive", api.Context.set_propagation) is set on every rank's context;
    all ranks must pass the same.  `view_selection` must be "off": the exchange carries each rank's top-n lists, not the
    per-view costs joint view selection needs (DESIGN.md §17)."""

    def __init__(self, scene, rank: int, world: int, device: int = 0, seed: int = 0xC0FFEE, group=None, options=None,
                 exchange: str = "nccl", propagation: str = "fixed", view_selection: str = "off", planar_prior=None):
        from . import api
        _check_exchange(exchange)
        api.check_propagation(propagation)
        _check_view_selection(view_selection)
        _check_planar_prior(planar_prior)
        self.scene, self.rank, self.world, self.group = scene, rank, world, group
        self.local = partition_views(scene.n_views, world)[rank]
        if not self.local:
            raise ValueError("more ranks than source views")
        self.ctx = api.Context(scene.cols, scene.rows, len(self.local), device=device)
        ctx = self.ctx
        for k, v in (options or {}).items():
            ctx.set_option(k, v)
        ctx.set_propagation(propagation)
        ctx.set_params(scene.params)
        self.upload(scene)
        ctx.set_rng(seed)
        uid = None
        if world > 1:
            import torch.distributed as dist
            box = [api.shard_unique_id() if rank == 0 else None]
            src = dist.get_global_rank(group, 0) if group is not None else 0
            dist.broadcast_object_list(box, src=src, group=group)
            uid = box[0]
        ctx.shard_comm_init(uid, rank, world)
        self.exchange = exchange if world > 1 else "none"
        self.collectives = 0

    def upload(self, scene, images=None):
        """(Re)upload the reference image and this rank's views; `images` may be a list of pinned host tensors."""
        imgs = scene.images if images is None else images
        get = (lambda i: np.ascontiguousarray(imgs[i])) if isinstance(imgs, np.ndarray) else (lambda i: imgs[i])
        self.ctx.set_reference(get(0), scene.cameras[0])
        for v, pos in enumerate(self.local):
            idx = scene.subset[pos]
            self.ctx.set_view(v, get(idx), scene.cameras[idx])
        self.ctx.set_num_views(len(self.local))

    def run_timed(self) -> float:
        """The sharded runcuda(); returns the sweep time in ms (reference's own span, max over ranks is the caller's job)."""
        ms = self.ctx.shard_run()
        self.collectives = self.ctx.stats()["collectives"]
        return ms

    def run(self):
        """runcuda() with sharded views: returns (norm4, cost) like Context.get_state after gpm_run."""
        self.run_timed()
        return self.ctx.get_state()

    def close(self):
        self.ctx.close()

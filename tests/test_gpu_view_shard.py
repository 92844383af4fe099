"""Source-view sharding (multi-GPU mode) on one GPU: the ranks are simulated by separate contexts holding disjoint
view subsets; the all-gather is a torch.cat.  The merged flow must reproduce the single-context run bit for bit.
(The NCCL exchange behind gpm_shard_run is exercised by test_gpu_view_shard_nccl.py when >= 2 GPUs are visible and by
tools/run_shard_nccl.py under torchrun; the host-side list merging by the gloo tests.)"""
import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu


def open_ranks(sc, world, seed=0xC0FFEE, options=None):
    """One context per rank of a shard group of `world` ranks, each holding its share of the source views."""
    from gipuma_b200 import multigpu as M
    from gipuma_b200 import api
    parts = M.partition_views(sc.n_views, world)
    ctxs = []
    for r in range(world):
        ctx = api.Context(sc.cols, sc.rows, len(parts[r]))
        for k, v in (options or {}).items():
            ctx.set_option(k, v)
        ctx.set_params(sc.params)
        ctx.set_reference(np.ascontiguousarray(sc.images[0]), sc.cameras[0])
        for v, pos in enumerate(parts[r]):
            ctx.set_view(v, np.ascontiguousarray(sc.images[sc.subset[pos]]), sc.cameras[sc.subset[pos]])
        ctx.set_num_views(len(parts[r]))
        ctx.set_rng(seed)
        ctxs.append(ctx)
    return ctxs


class SimulatedShard:
    """A shard group whose ranks are contexts on this GPU; the all-gather is a torch.cat."""

    def __init__(self, sc, world, seed=0xC0FFEE, options=None):
        self.world = world
        self.ctxs = open_ranks(sc, world, seed, options)
        self.n_stages = self.ctxs[0].shard_num_stages()

    def stage(self, colour, st, prev):
        """One exchange stage on every simulated rank: accept of the previous stage (fused) + evaluation; returns the
        rank-major concatenation of the lists, i.e. what an all-gather hands to every rank."""
        import torch
        n = self.ctxs[0].shard_stage_floats(st) if st < self.n_stages else 0
        locs = []
        for ctx in self.ctxs:
            buf = torch.empty(n, dtype=torch.float32, device="cuda") if n else None
            ctx.shard_stage(colour, st, prev, self.world, buf)
            locs.append(buf)
        torch.cuda.synchronize()
        return torch.cat(locs) if n else None

    def init(self):
        """Random planes, stage 0 and its accept; returns the gathered stage-0 lists."""
        for ctx in self.ctxs:
            ctx.init_planes()
        g0 = self.stage(0, 0, None)
        for ctx in self.ctxs:
            ctx.shard_finish_init(g0, self.world)
        return g0

    def colour(self, colour, after_stage=None):
        """Stages 1 .. n_stages - 1 of one colour and its closing accept (stage n_stages); after_stage(st, gathered) is
        called after each of them (gathered is None after the closing accept)."""
        prev = None
        for st in range(1, self.n_stages + 1):
            prev = self.stage(colour, st, prev)
            if after_stage is not None:
                after_stage(st, prev)

    def close(self):
        for ctx in self.ctxs:
            ctx.close()


def _sharded_run(sc, world, seed=0xC0FFEE):
    grp = SimulatedShard(sc, world, seed)
    grp.init()
    for _ in range(sc.params.iterations):
        for colour in (0, 1):
            grp.colour(colour)
    outs = []
    for ctx in grp.ctxs:
        ctx.finalize()
        outs.append(ctx.get_state())
    grp.close()
    return outs


@pytest.mark.parametrize("cfg,rows,cols,views,world,box,nbest", [
    (2, 64, 96, 6, 1, 15, 3),          # degenerate: one rank holds every view
    (2, 64, 96, 6, 2, 15, 3),
    (2, 96, 128, 10, 4, 11, 3),
    (4, 64, 96, 35, 2, 7, 3),          # > 32 views in total, 18 + 17 per rank
    (2, 64, 96, 3, 2, 9, 5),           # n_best larger than the number of views
])
def test_view_shard_equals_single_context(cfg, rows, cols, views, world, box, nbest):
    from gipuma_b200 import api, scene as S
    sc = S.make_config(cfg, rows=rows, cols=cols, n_views=views, iterations=2, seed=555)
    sc.params.box_hsize = sc.params.box_vsize = box
    sc.params.n_best = nbest
    single, _, _ = api.runcuda(sc, seed=0xC0FFEE)
    outs = _sharded_run(sc, world)
    for n4, c in outs:                                     # every rank ends with the same, identical state
        assert bits_equal(n4, single.norm4) == 0
        assert bits_equal(c, single.c) == 0


def test_view_shard_color_images():
    from gipuma_b200 import api, scene as S
    sc = S.colorize(S.make_config(2, rows=64, cols=96, n_views=5, iterations=2, seed=556))
    sc.params.box_hsize = sc.params.box_vsize = 9
    single, _, _ = api.runcuda(sc, seed=0xC0FFEE)
    for n4, c in _sharded_run(sc, 2):
        assert bits_equal(n4, single.norm4) == 0 and bits_equal(c, single.c) == 0


def test_view_shard_runner_single_rank_stream_ordered():
    """multigpu.ViewShardRunner at world size 1 = gpm_shard_run: the whole sharded flow enqueued on the context's stream behind
    the C-ABI, no host synchronisation in between — must equal the fused single-context run bit for bit."""
    from gipuma_b200 import api, multigpu as M, scene as S
    sc = S.make_config(4, rows=96, cols=128, n_views=12, iterations=2, seed=557)
    single, _, _ = api.runcuda(sc, seed=0xC0FFEE)
    run = M.ViewShardRunner(sc, 0, 1)
    for _ in range(2):                                     # twice: the second run re-uses buffers and memo state
        n4, c = run.run()
        assert bits_equal(n4, single.norm4) == 0 and bits_equal(c, single.c) == 0
    run.close()


def test_view_shard_refuses_other_combinations():
    import torch
    from gipuma_b200 import api, scene as S
    sc = S.make_config(1, rows=64, cols=96)
    sc.params.cost_comb = S.COMB_GOOD
    with api.Context(sc.cols, sc.rows, sc.n_views) as ctx:
        ctx.load_scene(sc)
        buf = torch.empty(ctx.shard_stage_floats(1), dtype=torch.float32, device="cuda")
        with pytest.raises(api.GipumaError):
            ctx.shard_stage(0, 1, None, 1, buf)

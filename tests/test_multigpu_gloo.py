"""Host-side multi-GPU logic on CPU: world-size-2 `gloo` process groups (no GPU in this container).

* reference-view batch: the round-robin assignment covers every reference view exactly once and the timing
  plumbing (barrier + MAX all-reduce, as bench.py does it) runs;
* source-view shard: per-rank local top-n lists, all-gathered and merged, reproduce the reference's
  best-n-over-all-views combination (pmCostMultiview_cu, gipuma.cu:770-805) of the UNsharded view costs — the
  NumPy functions used here are the host mirrors of the device functions `local_topn` / `shard_merge`.
"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from gipuma_b200 import multigpu as M


def reference_combine(costs, n_best):
    """Restatement of pmCostMultiview_cu's COMB_BEST_N tail (gipuma.cu:770-805) for one cost vector."""
    cv = [np.float32(c) if c < M.MAXCOST else np.float32(M.MAXCOST) for c in costs]
    num_valid = sum(1 for c in costs if c < M.MAXCOST)
    cv.sort()
    num_best = min(num_valid, n_best)
    cost = np.float32(0)
    for i in range(num_best):
        cost = np.float32(cost + cv[i])
    cost = np.float32(cost / np.float32(num_best)) if num_best else np.float32(M.MAXCOST)
    if cost != cost or cost > M.MAXCOST or cost < 0:
        cost = np.float32(M.MAXCOST)
    return cost


def test_partitions_cover_everything_once():
    for n in (1, 2, 9, 10, 47, 64):
        for world in (1, 2, 3, 4, 8):
            parts = M.partition_views(n, world)
            assert len(parts) == world and sorted(sum(parts, [])) == list(range(n))
            assert max(map(len, parts)) - min(map(len, parts)) <= 1
            refs = [M.assign_reference_views(n, r, world) for r in range(world)]
            assert sorted(sum(refs, [])) == list(range(n))


def test_merge_matches_reference_combination_single_process():
    rng = np.random.default_rng(3)
    for n_views, world, n_best in [(10, 2, 3), (47, 4, 3), (5, 4, 3), (3, 2, 5), (64, 8, 2)]:
        costs = rng.uniform(1, 60, size=(200, n_views)).astype(np.float32)
        costs[rng.uniform(size=costs.shape) < 0.05] = 1200.0                    # some views above MAXCOST
        costs[7] = 1500.0                                                        # a pixel with no valid view at all
        parts = M.partition_views(n_views, world)
        lists = np.stack([M.local_topn(costs[:, p], n_best) if p else np.full((200, n_best), np.inf, np.float32) for p in parts])
        lists[:, 11] = np.inf                                                    # a slot every rank skipped: no entry at all
        merged = M.merge_topn(lists, n_best)
        want = np.array([reference_combine(row, n_best) for row in costs], dtype=np.float32)
        want[11] = np.inf                                                        # never accepted, whatever the pixel's cost
        assert want[7] == np.float32(M.MAXCOST)
        assert np.array_equal(merged.view(np.uint32), want.view(np.uint32))


def test_hybrid_layout():
    group_of, rank_in, members = M.hybrid_layout(8, 4)
    assert group_of == [0, 0, 0, 0, 1, 1, 1, 1] and rank_in == [0, 1, 2, 3, 0, 1, 2, 3] and members == [[0, 1, 2, 3], [4, 5, 6, 7]]
    assert M.hybrid_layout(4, 1)[2] == [[0], [1], [2], [3]]
    with pytest.raises(ValueError):
        M.hybrid_layout(6, 4)
    # 8 GPUs, 2 groups: reference views 0..4 -> group 0 gets 0,2,4; group 1 gets 1,3
    assert M.assign_reference_views(5, 0, 2) == [0, 2, 4] and M.assign_reference_views(5, 1, 2) == [1, 3]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, n_views, n_best, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(11)                                             # same stream on all ranks
    costs = rng.uniform(1, 60, size=(300, 8, n_views)).astype(np.float32)       # [pixel, hypothesis slot, view]
    mine = M.partition_views(n_views, world)[rank]
    loc = torch.from_numpy(np.ascontiguousarray(M.local_topn(costs[..., mine], n_best))).reshape(-1)
    gat = torch.empty(world * loc.numel(), dtype=torch.float32)               # flat, rank-major — as ViewShardRunner does
    dist.all_gather_into_tensor(gat, loc)
    merged = M.merge_topn(gat.numpy().reshape(world, 300, 8, n_best), n_best)
    want = np.array([[reference_combine(costs[p, k], n_best) for k in range(8)] for p in range(300)], dtype=np.float32)
    ok = np.array_equal(merged.view(np.uint32), want.view(np.uint32))
    # every rank must hold the same merged result (state stays identical on all ranks)
    chk = torch.from_numpy(merged.copy())
    dist.all_reduce(chk, op=dist.ReduceOp.MAX)
    same = np.array_equal(chk.numpy().view(np.uint32), merged.view(np.uint32))
    # reference-view batch plumbing: barrier + max over ranks of a per-rank time
    dist.barrier()
    t = torch.tensor([10.0 + rank], dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    refs = M.assign_reference_views(5, rank, world)
    with open(os.path.join(out_dir, "r%d.txt" % rank), "w") as fh:
        fh.write("%d %d %.1f %s\n" % (ok, same, float(t), ",".join(map(str, refs))))
    dist.destroy_process_group()


@pytest.mark.parametrize("n_views,n_best", [(10, 3), (3, 3)])
def test_view_shard_merge_world2_gloo(tmp_path, n_views, n_best):
    world, port = 2, _free_port()
    mp.spawn(_worker, args=(world, port, n_views, n_best, str(tmp_path)), nprocs=world, join=True)
    seen = []
    for r in range(world):
        ok, same, tmax, refs = open(tmp_path / ("r%d.txt" % r)).read().split()
        assert ok == "1" and same == "1" and float(tmax) == 11.0
        seen += [int(x) for x in refs.split(",") if x]
    assert sorted(seen) == list(range(5))


def test_bench_sharded_layout_covers_every_view_once():
    """bench.py's view_shard / hybrid modes: every group's ranks together hold each source view exactly once, rank 0 is the one
    that also runs the unsharded comparison, and `--shard` must divide the world size."""
    import argparse
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("bench_module2", os.path.join(root, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    for world, mode, shard_opt, config, nviews in ((2, "auto", 0, 6, 60), (8, "auto", 0, 6, 60), (4, "view_shard", 0, 4, 47), (8, "hybrid", 4, 5, 64), (4, "hybrid", 0, 5, 64)):
        args = argparse.Namespace(mode=mode, config=config if mode != "auto" else 0, shard=shard_opt, color=False, neighbours=8, scene="smooth", no_check=False)
        m, cfg, shard = bench.resolve(args, world)
        assert cfg == config and world % shard == 0
        per_group = {}
        checks = 0
        for rank in range(world):
            group, rank_in, members, mine, check = bench.sharded_layout(args, cfg, shard, rank, world)
            per_group.setdefault(group, []).extend(mine)
            checks += int(check)
            assert rank in members[group] and members[group][rank_in] == rank
        assert checks == 1
        assert len(per_group) == world // shard
        for views in per_group.values():
            assert sorted(views) == list(range(nviews))
    with pytest.raises(SystemExit):
        bench.resolve(argparse.Namespace(mode="hybrid", config=0, shard=3, color=False, neighbours=8, scene="smooth"), 8)


def test_view_shard_refuses_the_removed_peer_memory_exchange():
    """exchange="p2p" fails before any context or process group is touched; "nccl" is the only exchange."""
    for call in (lambda: M.ViewShardRunner(None, 0, 2, exchange="p2p"), lambda: M.run_hybrid(None, 1, 0, 2, 2, exchange="p2p")):
        with pytest.raises(ValueError, match="peer-memory exchange was removed"):
            call()
    with pytest.raises(ValueError, match="NCCL only"):
        M.ViewShardRunner(None, 0, 2, exchange="mpi")

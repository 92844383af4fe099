#!/usr/bin/env python
"""Source-view shard over real GPUs (NCCL): torchrun --nproc-per-node N tools/run_shard_nccl.py [--config 4]
Rank 0 also runs the single-GPU job and checks that the sharded result is bit-identical; prints one JSON line."""
import argparse, json, os, sys, time
import numpy as np
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch
import torch.distributed as dist
from gipuma_b200 import scene as S, api, multigpu as M

ap = argparse.ArgumentParser()
ap.add_argument("--config", type=int, default=4)
ap.add_argument("--rows", type=int, default=None)
ap.add_argument("--cols", type=int, default=None)
ap.add_argument("--views", type=int, default=None)
ap.add_argument("--iters", type=int, default=None)
ap.add_argument("--hybrid", type=int, default=0, help="view-shard width; world/width groups take different reference views")
ap.add_argument("--refs", type=int, default=2)
ap.add_argument("--repeat", type=int, default=2)
ap.add_argument("--opt", nargs="*", default=[], help="gpm_set_option name=value pairs for the sharded contexts")
ap.add_argument("--propagation", default="fixed", choices=["fixed", "adaptive"], help="propagation mode of every context (view-shard mode)")
args = ap.parse_args()
rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
if args.hybrid:
    mk = lambda ref: S.make_config(args.config, rows=args.rows, cols=args.cols, n_views=args.views, iterations=args.iters, seed=1234 + 17 * ref)
    outs = {}
    times = M.run_hybrid(mk, args.refs, rank, world, args.hybrid, device=local, on_result=lambda ref, n4, c: outs.__setitem__(ref, (n4, c)))
    ok = True
    for ref, (n4, c) in outs.items():
        single, _, _ = api.runcuda(mk(ref), device=local)
        ok = ok and np.array_equal(n4.view(np.uint32), single.norm4.view(np.uint32)) and np.array_equal(c.view(np.uint32), single.c.view(np.uint32))
    t = torch.tensor([sum(times), float(ok)], dtype=torch.float64, device="cuda")
    if world > 1:
        tm = t.clone(); dist.all_reduce(tm, op=dist.ReduceOp.MAX); tn = t.clone(); dist.all_reduce(tn, op=dist.ReduceOp.MIN)
        t = torch.stack([tm[0], tn[1]])
    if rank == 0:
        print(json.dumps({"mode": "hybrid", "world": world, "shard": args.hybrid, "reference_views": args.refs, "wall_s": float(t[0]),
                          "all_groups_bit_identical_to_single_gpu": bool(t[1] > 0.5)}))
    if world > 1:
        dist.barrier(); dist.destroy_process_group()
    sys.exit(0)
sc = S.make_config(args.config, rows=args.rows, cols=args.cols, n_views=args.views, iterations=args.iters,
                   workers=max(1, min(32, len(os.sched_getaffinity(0)) // max(1, world))))
opts = {k: int(v) for k, v in (o.split("=") for o in args.opt)}
run = M.ViewShardRunner(sc, rank, world, device=local, options=opts, propagation=args.propagation)
run.run()                                              # warm-up (NCCL communicator, kernels)
torch.cuda.synchronize()
best, sweep = 1e30, 1e30
for _ in range(args.repeat):
    if world > 1:
        dist.barrier()
        torch.cuda.synchronize()
    t0 = time.perf_counter()
    ms = run.run_timed()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    tt = torch.tensor([dt, ms], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    best, sweep = min(best, float(tt[0])), min(sweep, float(tt[1]))
n4, c = run.ctx.get_state()
t = torch.tensor([best], dtype=torch.float64, device="cuda")
out = None
if rank == 0:
    with api.Context(sc.cols, sc.rows, sc.n_views, device=local) as one:
        one.load_scene(sc)
        one.set_propagation(args.propagation)
        one.run()
        ms = one.run()
        s4, s1 = one.get_state()
    same = np.array_equal(n4.view(np.uint32), s4.view(np.uint32)) and np.array_equal(c.view(np.uint32), s1.view(np.uint32))
    out = {"mode": "view_shard", "exchange": run.exchange, "opts": opts, "propagation": args.propagation, "config": sc.name, "rows": sc.rows, "cols": sc.cols, "views": sc.n_views, "world": world,
           "wall_s_incl_init": float(t), "sweep_ms_max_over_ranks": sweep, "single_over_sharded_sweep": ms / sweep, "mpixel_iters_per_s": sc.rows * sc.cols * sc.params.iterations / 1e6 / float(t),
           "single_gpu_sweep_ms": ms, "bit_identical_to_single_gpu": bool(same), "collectives": run.collectives}
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
if out:
    print(json.dumps(out))

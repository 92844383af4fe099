"""Per-launch k_sweep times of bench.py's single-GPU workload (BASELINE config 2: 1600x1200, 10 source views, box 15,
8 iterations) for several built trees, alternated in one session, and the sweep's fetch counts (DESIGN.md §5).

    python tools/share_bench.py --trees . /path/to/parent/tree [--repeats 3] [--count-lib lib.so] [--scene hard]

Each tree must hold a built gipuma_b200 (its libgipuma_b200.so).  Every measurement runs in a child process of its own:
one warm-up run, then one run under torch.profiler (CUDA activity only); the k_sweep kernels are listed in launch order.
`pairs` counts the (view, sample) pairs consumed by cost chains, i.e. fetches a per-pixel evaluation would make.  A
library compiled with -DGPM_SHARE_COUNT_FETCHES (--count-lib; the build recipe with that flag added) counts in `pairs` the
(view, texel) pairs really fetched, and in the stats' last slot the plane-major pass's share of the usual `pairs`.
Prints the GPU's name and power limit, one table per tree and one JSON line."""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def child(tree, lib, scene, out):
    sys.path.insert(0, os.path.abspath(tree))
    import ctypes as C
    import torch
    from torch.profiler import ProfilerActivity, profile
    from gipuma_b200 import api, scene as S
    if lib:
        api.LIB_PATH = os.path.abspath(lib)
    sc = S.make_config(2, seed=1234, hard=(scene == "hard"))
    with api.Context(sc.cols, sc.rows, sc.n_views) as ctx:
        ctx.load_scene(sc)
        ctx.run()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ms = ctx.run()
            torch.cuda.synchronize()
        raw = (C.c_ulonglong * 8)()
        ctx._check(ctx.lib.gpm_get_stats(ctx.h, raw))
        st = ctx.stats()
        n4, c = ctx.get_state()
    sweeps = [e for e in prof.events() if e.device_type.name == "CUDA" and "k_sweep" in e.name]
    sweeps.sort(key=lambda e: e.time_range.start)
    res = {"tree": tree, "run_ms": ms, "k_sweep_us": [round(e.time_range.elapsed_us(), 1) for e in sweeps],
           "pairs": st["pairs"], "hypotheses": st["hypotheses"], "pass_pairs": int(raw[7]) if lib else None,
           "digest": int((n4.view("uint32").astype("uint64").sum() + c.view("uint32").astype("uint64").sum()) % (1 << 61))}
    with open(out, "w") as fh:
        json.dump(res, fh)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", nargs="+", default=[ROOT])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--count-lib", default=None, help="a library built with -DGPM_SHARE_COUNT_FETCHES, run with the first tree")
    ap.add_argument("--scene", default="smooth", choices=["smooth", "hard"])
    ap.add_argument("--child", nargs=3, metavar=("TREE", "LIB", "OUT"))
    a = ap.parse_args()
    if a.child:
        return child(a.child[0], a.child[1] if a.child[1] != "-" else None, a.scene, a.child[2])
    import tempfile
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("GPU:", q.stdout.strip())
    runs = {t: [] for t in a.trees}
    with tempfile.TemporaryDirectory() as tmp:
        jobs = [(t, "-") for _ in range(a.repeats) for t in a.trees] + ([(a.trees[0], a.count_lib)] if a.count_lib else [])
        for i, (t, lib) in enumerate(jobs):
            out = os.path.join(tmp, "%d.json" % i)
            subprocess.run([sys.executable, __file__, "--scene", a.scene, "--child", t, lib, out], check=True)
            with open(out) as fh:
                runs[t].append(json.load(fh))
    summary = {}
    for t, rs in runs.items():
        timed = [r for r in rs if r["pass_pairs"] is None]
        per_launch = [min(x) for x in zip(*[r["k_sweep_us"] for r in timed])]
        print("\n%s: %d k_sweep launches, min over %d runs (us):" % (t, len(per_launch), len(timed)))
        print("  " + " ".join("%.0f" % v for v in per_launch))
        print("  sum %.1f ms, run %s ms, pairs %d, hypotheses %d, digest %d" %
              (sum(per_launch) / 1e3, [round(r["run_ms"], 1) for r in timed], timed[0]["pairs"], timed[0]["hypotheses"], timed[0]["digest"]))
        counted = [r for r in rs if r["pass_pairs"] is not None]
        if counted:
            c, logical = counted[0], timed[0]["pairs"]
            real_pass = c["pairs"] - (logical - c["pass_pairs"])
            print("  counting build: pairs %d, of which the plane-major pass %d; really fetched %d, of which the pass %d: "
                  "%.3fx fewer in all, %.3fx fewer in the pass" % (logical, c["pass_pairs"], c["pairs"], real_pass,
                                                                  logical / c["pairs"], c["pass_pairs"] / max(1, real_pass)))
        summary[t] = {"k_sweep_us": per_launch, "sum_ms": sum(per_launch) / 1e3, "run_ms": [r["run_ms"] for r in timed],
                      "pairs": timed[0]["pairs"], "hypotheses": timed[0]["hypotheses"], "digest": timed[0]["digest"],
                      "counted": counted[0] if counted else None}
    print(json.dumps({"gpu": q.stdout.strip(), "scene": a.scene, "trees": summary}))


if __name__ == "__main__":
    main()

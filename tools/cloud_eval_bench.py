"""Time the point-cloud distances (gpm_nearest_dist) at the DTU size against scipy's cKDTree and print one JSON line.

    python tools/cloud_eval_bench.py [--views 49] [--rows 1200] [--cols 1600] [--stride 3] [--reps 5] [--hole 25]

Workloads, max_dist 20 (mm), both directions (accuracy: reconstruction -> ground truth; completeness: the reverse):
  full   the ground-truth-fused cloud of the first `--views` DTU cameras (gpm_fuse of scene.render_norm4, the scripts'
         options) against scene.gt_points of the same maps, every `--stride`-th row and column;
  holed  the same with every vertex within `--hole` mm of a seeded vertex removed, so that the ground-truth points in the
         hole search out to the cap.
gpm_nearest_dist is timed with its own CUDA events (upload_ms, build_ms, query_ms), median of `--reps` calls after one
warm-up call.  The CPU baseline is cKDTree on the same task, build plus query(k=1, distance_upper_bound=max_dist), with 1
worker and with every host core, timed once each.  A seeded sample of `--check` queries per direction is compared with the
certified restatement (oracle/pycloud.py).  Needs a CUDA device; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MAX_DIST = 20.0


def _kdtree(q, b, workers):
    from scipy.spatial import cKDTree
    t0 = time.perf_counter()
    tree = cKDTree(b)
    t1 = time.perf_counter()
    tree.query(q, k=1, distance_upper_bound=MAX_DIST, workers=workers)
    t2 = time.perf_counter()
    return {"build_s": round(t1 - t0, 3), "query_s": round(t2 - t1, 3), "total_s": round(t2 - t0, 3)}


def _direction(q, b, reps, check, rng):
    from gipuma_b200 import api
    from oracle import pycloud
    api.nearest_distance(q, b, MAX_DIST)
    runs = [api.nearest_distance(q, b, MAX_DIST) for _ in range(reps)]
    assert all(r[0].tobytes() == runs[0][0].tobytes() for r in runs), "distances are not deterministic"
    med = {k: float(np.median([r[1][k] for r in runs])) for k in ("upload_ms", "build_ms", "query_ms")}
    pick = np.sort(rng.choice(len(q), min(check, len(q)), replace=False))
    want, _ = pycloud.certified(q[pick], b, MAX_DIST)
    d = runs[0][0]
    gpu_s = (med["build_ms"] + med["query_ms"]) * 1e-3
    out = {"n_query": len(q), "n_data": len(b), **{k: round(v, 2) for k, v in med.items()},
           "queries_per_s": round(len(q) / gpu_s, 0), "cell_size": round(runs[0][1]["cell_size"], 4),
           "n_cells": runs[0][1]["n_cells"], "share_inf": round(float(np.isinf(d).mean()), 5),
           "sample_exact": bool(d[pick].tobytes() == want.tobytes()), "sample": len(pick)}
    q64, b64 = q.astype(np.float64), b.astype(np.float64)
    out["ckdtree_1_worker"] = _kdtree(q64, b64, 1)
    out["ckdtree_all_cores"] = _kdtree(q64, b64, -1)
    out["gpu_speedup_vs_all_cores"] = round(out["ckdtree_all_cores"]["total_s"] / gpu_s, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--rows", type=int, default=1200)
    ap.add_argument("--cols", type=int, default=1600)
    ap.add_argument("--stride", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--hole", type=float, default=25.0)
    ap.add_argument("--check", type=int, default=20000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("cloud_eval_bench: needs a CUDA device")
    from gipuma_b200 import api, scene as S
    Ps = [S.load_dtu_projections()[i] for i in range(a.views)]
    scale = 1600.0 / a.cols
    hf = S.HeightField(z0=550.0, unit=550.0 / S.prepare_cameras(Ps[:1], scale)[0].fx, seed=77)
    maps = S.render_norm4(Ps, scale, a.rows, a.cols, hf)
    prm = dict(depth_min=300.0, depth_max=800.0, disp_thresh=0.1, normal_thresh=30.0, num_consistent=3)   # scripts/dtu_fast.sh
    v, _ = api.fuse(maps, Ps, cam_scale=scale, **prm)
    gt = S.gt_points(Ps, scale, a.rows, a.cols, hf, stride=a.stride, norm4=maps)
    del maps
    rec = np.ascontiguousarray(np.stack([v["x"], v["y"], v["z"]], axis=1))
    rng = np.random.default_rng(2026)
    centre = rec[rng.integers(len(rec))]
    holed = np.ascontiguousarray(rec[((rec - centre) ** 2).sum(1) > a.hole ** 2])
    gpu = {"name": torch.cuda.get_device_name(0)}
    try:
        gpu["power_limit_w"] = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        gpu["power_limit_w"] = "unknown (%s)" % e
    out = {"workload": "cloud distances, %d views %dx%d: GT-fused cloud vs gt_points stride %d, max_dist %g"
                       % (a.views, a.cols, a.rows, a.stride, MAX_DIST), "gpu": gpu, "host_cores": os.cpu_count() or 0,
           "hole_mm": a.hole, "holed_removed": len(rec) - len(holed)}
    for name, r in (("full", rec), ("holed", holed)):
        out[name] = {"accuracy": _direction(r, gt, a.reps, a.check, rng), "completeness": _direction(gt, r, a.reps, a.check, rng)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

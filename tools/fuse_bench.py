"""Time the depth-map fusion (gpm_fuse) at the DTU size and print one JSON line.

    python tools/fuse_bench.py [--views 49] [--rows 1200] [--cols 1600] [--reps 5] [--oracle-passes 1]

Input: ground-truth norm4 maps of the first `--views` DTU cameras looking at a seeded height field (scene.render_norm4), so
the case does not depend on a PatchMatch run.  gpm_fuse is timed with its own CUDA events (`fuse_ms`: first fusion kernel to
the last vertex download, host inputs already uploaded; `upload_ms`: the host-to-device copies before it), after one warm-up
call, median of `--reps` calls.  The single-thread C restatement (oracle/fusion_oracle.c) is timed on the first
`--oracle-passes` reference views only; its time per pass is not the GPU's, whose passes get cheaper as pixels are used.
Needs a CUDA device; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--rows", type=int, default=1200)
    ap.add_argument("--cols", type=int, default=1600)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-passes", type=int, default=1)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("fuse_bench: needs a CUDA device")
    from gipuma_b200 import api, scene as S
    from oracle import pyfusion
    Ps = [S.load_dtu_projections()[i] for i in range(a.views)]
    scale = 1600.0 / a.cols
    hf = S.HeightField(z0=550.0, unit=550.0 / S.prepare_cameras(Ps[:1], scale)[0].fx, seed=77)
    gt = S.render_norm4(Ps, scale, a.rows, a.cols, hf)
    prm = dict(depth_min=300.0, depth_max=800.0, disp_thresh=0.1, normal_thresh=30.0, num_consistent=3)   # scripts/dtu_fast.sh
    api.fuse(gt, Ps, cam_scale=scale, **prm)
    runs = [api.fuse(gt, Ps, cam_scale=scale, **prm) for _ in range(a.reps)]
    fuse_ms = sorted(r[1]["fuse_ms"] for r in runs)
    upload_ms = sorted(r[1]["upload_ms"] for r in runs)
    assert all(r[0].tobytes() == runs[0][0].tobytes() for r in runs), "fusion is not deterministic"
    t0 = time.perf_counter()
    ov, _, _ = pyfusion.fuse(gt, api.fuse_cameras(Ps, scale), refs=(0, a.oracle_passes), threads=1, **prm)
    oracle_s = time.perf_counter() - t0
    k = int((runs[0][1]["source"][:, 0] < a.oracle_passes).sum())
    assert k == len(ov) and runs[0][0][:k].tobytes() == ov.tobytes(), "GPU and C restatement differ"
    gpu = {"name": torch.cuda.get_device_name(0)}
    try:
        gpu["power_limit_w"] = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        gpu["power_limit_w"] = "unknown (%s)" % e
    med = fuse_ms[len(fuse_ms) // 2]
    print(json.dumps({
        "workload": "fuse %d views %dx%d ground truth" % (a.views, a.cols, a.rows), "gpu": gpu,
        "vertices": len(runs[0][0]), "fuse_ms": round(med, 2), "fuse_ms_all": [round(x, 2) for x in fuse_ms],
        "upload_ms": round(upload_ms[len(upload_ms) // 2], 2),
        "mpixel_views_per_s": round(a.views * a.rows * a.cols / (med * 1e-3) / 1e6, 1),
        "oracle_1thread_s": round(oracle_s, 2), "oracle_passes": a.oracle_passes, "oracle_vertices": len(ov),
        "host_cores": os.cpu_count() or 0}))


if __name__ == "__main__":
    main()

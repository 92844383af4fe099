"""Fused-cloud quality and sweep time of the geometric-consistency pass (DESIGN.md §14) against photometric PatchMatch alone,
with the same total number of iterations; prints one JSON line.

    python tools/geo_bench.py [--rows 600] [--cols 800] [--cams 16] [--iterations 6] [--geo-iterations 2]
                              [--configs 0.1:2,0.2:3,0.5:3] [--scenes smooth,hard]

Scenes: the textured height field seen by the first `--cams` DTU cameras at `--cols` x `--rows` (K scaled from
1600 x 1200), and its hard variant (occluding blocks, a texture-less band, sensor noise).  Every second camera is a
reference view; parameters: box 11, n_best 3, depth 300..800, views at 5..45 degrees, at most 6 per reference.
  photometric   batch_run with `--iterations` iterations;
  geometric     geometric_pass: `--iterations` - `--geo-iterations` photometric iterations, then `--geo-iterations` with the
                geometric term, for each weight:max_err of `--configs`.
Each output is fused (gpm_fuse, depth 300..800, disparity 0.1, normals 30 degrees, 2 consistent views) and scored with
evaluate_cloud against the scene's ground-truth points (max_dist 10 units, taus 0.25 / 0.5 / 1 unit; a unit is one
reference pixel at the mean depth).  Sweep time per iteration: host time of each view's sweep call (which ends in a
stream synchronisation) over its iterations, median over the views, for pass 1 (photometric) and pass 2 (geometric) of the
same runs.  Needs a CUDA device; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600)
    ap.add_argument("--cols", type=int, default=800)
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--iterations", type=int, default=6)
    ap.add_argument("--geo-iterations", type=int, default=2)
    ap.add_argument("--configs", default="0.1:2,0.2:3,0.5:3")
    ap.add_argument("--scenes", default="smooth,hard")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("geo_bench: needs a CUDA device")
    from gipuma_b200 import api, scene as S
    gpu = {"name": torch.cuda.get_device_name(0)}
    try:
        gpu["power_limit_w"] = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        gpu["power_limit_w"] = "unknown (%s)" % e
    configs = [tuple(float(x) for x in c.split(":")) for c in a.configs.split(",")]
    Ps = [S.load_dtu_projections()[i] for i in range(a.cams)]
    scale = 1600.0 / a.cols
    refs = list(range(0, a.cams, 2))
    fPs = [Ps[r] for r in refs]
    kw = dict(cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
    fuse_kw = dict(depth_min=300.0, depth_max=800.0, disp_thresh=0.1, normal_thresh=30.0, num_consistent=2)
    out = {"workload": "%d DTU cameras at %dx%d, %d reference views, %d iterations in all" % (a.cams, a.cols, a.rows, len(refs), a.iterations),
           "gpu": gpu, "geo_iterations": a.geo_iterations}

    def params(iterations):
        p = S.AlgorithmParameters(box_hsize=11, box_vsize=11, iterations=iterations, n_best=3, cost_comb=S.COMB_BEST_N, gamma=10.0)
        p.depthMin, p.depthMax = 300.0, 800.0
        return p

    for scene in a.scenes.split(","):
        cams = S.prepare_cameras(Ps, scale)
        hf = S.HeightField(z0=550.0, unit=550.0 / cams[0].fx, seed=77, hard=scene == "hard")
        images = np.stack([S.render_view(c, a.rows, a.cols, hf, noise_seed=(1000 + i) if hf.hard else None)[0]
                           for i, c in enumerate(cams)])
        gt = S.gt_points(fPs, scale, a.rows, a.cols, hf, stride=2)
        unit = hf.unit
        taus = (0.25 * unit, 0.5 * unit, unit)

        def score(n4):
            v, _ = api.fuse(n4, fPs, cam_scale=scale, **fuse_kw)
            s = api.evaluate_cloud(v, gt, max_dist=10 * unit, taus=taus)
            return {"vertices": len(v), "accuracy_mean_units": round(s["accuracy_mean"] / unit, 4),
                    "completeness_mean_units": round(s["completeness_mean"] / unit, 4),
                    "f_score": [round(f, 4) for f in s["f_score"]]}

        res = {"unit": unit, "gt_points": len(gt)}
        n4, _, st = api.batch_run(images, Ps, params(a.iterations), refs, **kw)
        res["photometric"] = score(n4)
        for w, m in configs:
            n4, _, info = api.geometric_pass(images, Ps, params(a.iterations - a.geo_iterations), refs,
                                             geo_iterations=a.geo_iterations, weight=w, max_err=m, **kw)
            r = score(n4)
            r["pass1_ms_per_iteration"] = round(1e3 * float(np.median(info["pass1_sweep_s"])) / (a.iterations - a.geo_iterations), 3)
            r["pass2_ms_per_iteration"] = round(1e3 * float(np.median(info["pass2_sweep_s"])) / a.geo_iterations, 3)
            res["geometric w=%g max_err=%g" % (w, m)] = r
        out[scene] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()

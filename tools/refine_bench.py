"""Fused-cloud quality and sweep time of ACMH's refinement against Gipuma's (DESIGN.md §23); prints one JSON line.

    python tools/refine_bench.py [--rows 600] [--cols 800] [--cams 16] [--scenes smooth,hard,lit] [--costs pm,ncc]
                                 [--levels 2] [--perturbations 0.02]

Workload: ms_bench.py's (the first `--cams` DTU cameras at `--cols` x `--rows`, every second camera a reference view, box 11,
n_best 3, depth 300..800, views at 5..45 degrees, at most 6 per reference; the same fusion and evaluate_cloud set-up; scenes
smooth, hard and lit).  Per scene and cost, each flow runs once with refinement "gipuma" and once with "acmh" at each of
`--perturbations`: batch_run with 6 iterations, geometric_pass with 4 + 2 and multiscale_pass with 4 photometric
iterations at the coarsest level and 2 with the geometric term at every level, at each of `--levels`.  Each row has the
F-score at 0.25, 0.5 and 1 unit, mean accuracy and completeness (units), vertices and the sweep ms summed over every view
(and level), CUDA events on gpm_stream; on the hard scene also the scores on its texture-less band (ms_bench.py's rule).
The GPU's name and power limit are read in the same run.  Needs a CUDA device; there is no CPU path.
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
    ap.add_argument("--scenes", default="smooth,hard,lit")
    ap.add_argument("--costs", default="pm,ncc")
    ap.add_argument("--levels", default="2")
    ap.add_argument("--perturbations", default="0.02")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("refine_bench: needs a CUDA device")
    from gipuma_b200 import api, scene as S
    gpu = {"name": torch.cuda.get_device_name(0)}
    try:
        gpu["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.split()
    except Exception as e:      # noqa: BLE001
        gpu["power_limit_w"] = "unknown (%s)" % e

    def log(msg):
        print("refine_bench: %s" % msg, file=sys.stderr, flush=True)

    levels = [int(x) for x in a.levels.split(",") if x]
    refinements = [("gipuma", None)] + [("acmh eps=%g" % float(e), {"kind": "acmh", "perturbation": float(e)})
                                        for e in a.perturbations.split(",") if e]
    out = {"gpu": gpu, "workload": "%d DTU cameras at %dx%d" % (a.cams, a.cols, a.rows)}
    costs = {"pm": {}, "ncc": dict(photometric="ncc", ncc_min_std=api.NCC_MIN_STD)}
    costs = {k: costs[k] for k in a.costs.split(",") if k}

    def params(iterations):
        p = S.AlgorithmParameters(box_hsize=11, box_vsize=11, iterations=iterations, n_best=3, cost_comb=S.COMB_BEST_N, gamma=10.0)
        p.depthMin, p.depthMax = 300.0, 800.0
        return p

    Ps = [S.load_dtu_projections()[i] for i in range(a.cams)]
    scale = 1600.0 / a.cols
    refs = list(range(0, a.cams, 2))
    fPs = [Ps[r] for r in refs]
    kw = dict(cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
    fuse_kw = dict(depth_min=300.0, depth_max=800.0, disp_thresh=0.1, normal_thresh=30.0, num_consistent=2)
    for scene in [x for x in a.scenes.split(",") if x]:
        log("%s: rendering" % scene)
        cams = S.prepare_cameras(Ps, scale)
        hf = S.HeightField(z0=550.0, unit=550.0 / cams[0].fx, seed=77, hard=scene == "hard")
        images = np.stack([S.render_view(c, a.rows, a.cols, hf, noise_seed=(1000 + i) if hf.hard else None)[0]
                           for i, c in enumerate(cams)]).astype(np.float32)
        if scene == "lit":
            rng = np.random.default_rng(2024)
            images = np.clip(np.stack([rng.uniform(0.6, 1.4) * im + rng.uniform(-40, 40) for im in images]), 0, 255).astype(np.float32)
        gt = S.gt_points(fPs, scale, a.rows, a.cols, hf, stride=2)
        unit = hf.unit
        in_band = lambda p: np.abs(p[:, 1] - 180.0 * unit) < 70.0 * unit          # noqa: E731  (HeightField's band rule)

        def score(n4, sweep_ms):
            v, _ = api.fuse(n4, fPs, cam_scale=scale, **fuse_kw)
            s = api.evaluate_cloud(v, gt, max_dist=10 * unit, taus=(0.25 * unit, 0.5 * unit, unit))
            r = {"f_score": [round(f, 4) for f in s["f_score"]], "accuracy_mean_units": round(s["accuracy_mean"] / unit, 4),
                 "completeness_mean_units": round(s["completeness_mean"] / unit, 4), "vertices": len(v),
                 "sweep_ms_total": round(sweep_ms, 1)}
            if scene == "hard":
                v = np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float32)
                b = api.evaluate_cloud(np.ascontiguousarray(v[in_band(v)]), np.ascontiguousarray(gt[in_band(gt)]),
                                       max_dist=10 * unit, taus=(unit,))
                r["band_f_score_1unit"] = round(b["f_score"][0], 4)
                r["band_completeness_mean_units"] = round(b["completeness_mean"] / unit, 4)
            return r

        res = {}
        for cost, photo in costs.items():
            row = {}
            for name, ref in refinements:
                n4, _, st = api.batch_run(images, Ps, params(6), refs, refinement=ref, **kw, **photo)
                row["batch_run 6, %s" % name] = score(n4, st["sweep_ms_total"])
                n4, _, info = api.geometric_pass(images, Ps, params(4), refs, geo_iterations=2, refinement=ref, **kw, **photo)
                row["geometric_pass 4 + 2, %s" % name] = score(n4, 1e3 * (sum(info["pass1_sweep_s"]) + sum(info["pass2_sweep_s"])))
                for L in levels:
                    n4, _, info = api.multiscale_pass(images, Ps, params(4), refs, levels=L, geo_iterations=2, refinement=ref,
                                                      **kw, **photo)
                    row["multiscale_pass levels %d, %s" % (L, name)] = score(n4, 1e3 * sum(info["level_sweep_s"]))
                log("%s %s %s: %s" % (scene, cost, name, {k: v for k, v in row.items() if k.endswith(name)}))
            res[cost] = row
        out[scene] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()

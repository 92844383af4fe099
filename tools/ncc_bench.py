"""Fused-cloud quality and sweep speed of the NCC photometric cost (DESIGN.md §15) against the reference's PM cost; prints one
JSON line.

    python tools/ncc_bench.py [--rows 600] [--cols 800] [--cams 16] [--iterations 6] [--geo-iterations 2]
                              [--min-std 1,2,4] [--scenes smooth,hard,lit] [--speed-iterations 4]

Quality: tools/geo_bench.py's set-up (the first `--cams` DTU cameras at `--cols` x `--rows`, every second camera a reference
view, box 11, n_best 3, depth 300..800, views at 5..45 degrees, at most 6 per reference; fusion with disparity 0.1, normals
30 degrees, 2 consistent views; evaluate_cloud against ground-truth points at stride 2, max_dist 10 units).  Scenes: the
smooth height field, its hard variant, and "lit": the smooth scene with a seeded per-view gain in [0.6, 1.4] and offset in
[-40, 40] applied to every image, clipped to [0, 255] (the share of clipped pixels is reported).  Per scene: PM and NCC at each
`--min-std`, photometric only (batch_run, `--iterations`) and with the geometric pass (geometric_pass, `--iterations` -
`--geo-iterations` photometric iterations, then `--geo-iterations` geometric ones, api.GEO_WEIGHT / GEO_MAX_ERR).
Speed: sweep ms per iteration from CUDA events on gpm_stream around gpm_sweep(`--speed-iterations`) after gpm_init and a
one-iteration warm-up, PM against NCC (min_std api.NCC_MIN_STD), at bench config 2's shape (1600 x 1200, 10 views, box 15)
and at 800 x 600, with gpm_get_stats' evaluated (view, sample) pairs and hypotheses of the timed sweep.  Needs a CUDA
device; there is no CPU path.
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
    ap.add_argument("--min-std", default="1,2,4")
    ap.add_argument("--scenes", default="smooth,hard,lit")
    ap.add_argument("--speed-iterations", type=int, default=4)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ncc_bench: needs a CUDA device")
    from gipuma_b200 import api, scene as S
    gpu = {"name": torch.cuda.get_device_name(0)}
    try:
        gpu["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.split()
    except Exception as e:      # noqa: BLE001
        gpu["power_limit_w"] = "unknown (%s)" % e

    def log(msg):
        print("ncc_bench: %s" % msg, file=sys.stderr, flush=True)

    out = {"gpu": gpu, "workload": "%d DTU cameras at %dx%d, %d iterations (geometric: last %d)" %
           (a.cams, a.cols, a.rows, a.iterations, a.geo_iterations)}
    stds = [float(x) for x in a.min_std.split(",")]
    Ps = [S.load_dtu_projections()[i] for i in range(a.cams)]
    scale = 1600.0 / a.cols
    refs = list(range(0, a.cams, 2))
    fPs = [Ps[r] for r in refs]
    kw = dict(cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
    fuse_kw = dict(depth_min=300.0, depth_max=800.0, disp_thresh=0.1, normal_thresh=30.0, num_consistent=2)

    def params(iterations):
        p = S.AlgorithmParameters(box_hsize=11, box_vsize=11, iterations=iterations, n_best=3, cost_comb=S.COMB_BEST_N, gamma=10.0)
        p.depthMin, p.depthMax = 300.0, 800.0
        return p

    for scene in [x for x in a.scenes.split(",") if x]:                    # --scenes "": speed only
        log("%s: rendering" % scene)
        cams = S.prepare_cameras(Ps, scale)
        hf = S.HeightField(z0=550.0, unit=550.0 / cams[0].fx, seed=77, hard=scene == "hard")
        images = np.stack([S.render_view(c, a.rows, a.cols, hf, noise_seed=(1000 + i) if hf.hard else None)[0]
                           for i, c in enumerate(cams)]).astype(np.float32)
        res = {}
        if scene == "lit":
            rng = np.random.default_rng(2024)
            lit = np.stack([rng.uniform(0.6, 1.4) * im + rng.uniform(-40, 40) for im in images])
            res["clipped_share"] = round(float(((lit < 0) | (lit > 255)).mean()), 4)
            images = np.clip(lit, 0, 255).astype(np.float32)
        gt = S.gt_points(fPs, scale, a.rows, a.cols, hf, stride=2)
        unit = hf.unit

        def score(n4):
            v, _ = api.fuse(n4, fPs, cam_scale=scale, **fuse_kw)
            s = api.evaluate_cloud(v, gt, max_dist=10 * unit, taus=(0.25 * unit, 0.5 * unit, unit))
            return {"vertices": len(v), "accuracy_mean_units": round(s["accuracy_mean"] / unit, 4),
                    "completeness_mean_units": round(s["completeness_mean"] / unit, 4), "f_score": [round(f, 4) for f in s["f_score"]]}

        for name, photo in [("pm", {})] + [("ncc min_std=%g" % s, dict(photometric="ncc", ncc_min_std=s)) for s in stds]:
            n4, _, _ = api.batch_run(images, Ps, params(a.iterations), refs, **kw, **photo)
            res[name] = {"photometric": score(n4)}
            n4, _, _ = api.geometric_pass(images, Ps, params(a.iterations - a.geo_iterations), refs, geo_iterations=a.geo_iterations,
                                          **kw, **photo)
            res[name]["with_geometric"] = score(n4)
            log("%s %s: %s" % (scene, name, res[name]))
        out[scene] = res

    speed = {}
    for rows, cols in ((1200, 1600), (600, 800)):
        sc = S.make_config(2, rows=rows, cols=cols, n_views=10, iterations=1, seed=7)
        sc.params.box_hsize = sc.params.box_vsize = 15
        row = {}
        for name in ("pm", "ncc"):
            with api.Context(cols, rows, len(sc.subset)) as ctx:
                ctx.load_scene(sc)
                if name == "ncc":
                    ctx.set_photometric("ncc", api.NCC_MIN_STD)
                ctx.init()
                ctx.sweep(1)
                stream = torch.cuda.ExternalStream(ctx.stream)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ctx.reset_stats()
                e0.record(stream)
                ctx.sweep(a.speed_iterations)
                e1.record(stream)
                e1.synchronize()
                st = ctx.stats()
                row[name] = {"ms_per_iteration": round(e0.elapsed_time(e1) / a.speed_iterations, 3), "pairs": st["pairs"],
                             "pairs_full": st["pairs_full"], "hypotheses": st["hypotheses"], "pruned": st["pruned"]}
        row["ncc_over_pm"] = round(row["ncc"]["ms_per_iteration"] / row["pm"]["ms_per_iteration"], 3)
        speed["%dx%d, 10 views, box 15" % (cols, rows)] = row
        log("speed %dx%d: %s" % (cols, rows, row))
    out["speed"] = speed
    print(json.dumps(out))


if __name__ == "__main__":
    main()

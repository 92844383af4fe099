"""Fused-cloud quality and sweep time of the geometric-consistency pass (DESIGN.md §14) against photometric PatchMatch alone,
with the same total number of iterations; prints one JSON line.

    python tools/geo_bench.py [--rows 600] [--cols 800] [--cams 16] [--iterations 6] [--geo-iterations 2]
                              [--configs 0.1:2,0.2:3,0.5:3] [--scenes smooth,hard] [--devices 0 [0,0 ...]] [--preset dtu]

Scenes: the textured height field seen by the first `--cams` DTU cameras at `--cols` x `--rows` (K scaled from
1600 x 1200), and its hard variant (occluding blocks, a texture-less band, sensor noise).  Every second camera is a
reference view; parameters: box 11, n_best 3, depth 300..800, views at 5..45 degrees, at most 6 per reference.
  photometric   batch_run with `--iterations` iterations;
  geometric     geometric_pass: `--iterations` - `--geo-iterations` photometric iterations, then `--geo-iterations` with the
                geometric term, for each weight:max_err of `--configs`.
Each output is fused (gpm_fuse, depth 300..800, disparity 0.1, normals 30 degrees, 2 consistent views) and scored with
evaluate_cloud against the scene's ground-truth points (stride 2, max_dist 10 units, taus 0.25 / 0.5 / 1 unit; a unit is one
reference pixel at the mean depth).
`--preset dtu`: the DTU size instead: 49 cameras at 1600 x 1200, every camera a reference view, the smooth scene, the
defaults api.GEO_WEIGHT:api.GEO_MAX_ERR only, fused with the DTU script's options (3 consistent views) and scored against
ground-truth points at stride 3.
`--devices`: one or more worker sets, each a comma-separated list of CUDA ordinals (one worker thread and context per entry;
a device may be listed twice); every run of every configuration is repeated for each set, and the outputs of later sets
must equal the first set's bit for bit.  When more than one GPU is visible, a set of all of them is added.  Per set: wall
time of the whole batch_run / geometric_pass call (after a one-iteration warm-up on every listed device), and sweep time per
iteration: CUDA-event time of each view's sweep call over its iterations, median over the views, for pass 1 (photometric)
and pass 2 (geometric).  Needs a CUDA device; there is no CPU path.
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
    ap.add_argument("--rows", type=int, default=600)
    ap.add_argument("--cols", type=int, default=800)
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--iterations", type=int, default=6)
    ap.add_argument("--geo-iterations", type=int, default=2)
    ap.add_argument("--configs", default="0.1:2,0.2:3,0.5:3")
    ap.add_argument("--scenes", default="smooth,hard")
    ap.add_argument("--devices", nargs="+", default=["0"])
    ap.add_argument("--preset", choices=["dtu"], default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("geo_bench: needs a CUDA device")
    from gipuma_b200 import api, scene as S
    gpu = {"name": torch.cuda.get_device_name(0), "visible": torch.cuda.device_count()}
    try:
        gpu["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.split()
    except Exception as e:      # noqa: BLE001
        gpu["power_limit_w"] = "unknown (%s)" % e
    fuse_kw = dict(depth_min=300.0, depth_max=800.0, disp_thresh=0.1, normal_thresh=30.0, num_consistent=2)
    stride = 2
    if a.preset == "dtu":
        a.rows, a.cols, a.cams, a.scenes = 1200, 1600, 49, "smooth"
        a.configs = "%g:%g" % (api.GEO_WEIGHT, api.GEO_MAX_ERR)
        fuse_kw["num_consistent"] = 3                                           # scripts/dtu_fast.sh
        stride = 3
    device_sets = [[int(x) for x in s.split(",")] for s in a.devices]
    if torch.cuda.device_count() > 1:
        device_sets.append(list(range(torch.cuda.device_count())))
    configs = [tuple(float(x) for x in c.split(":")) for c in a.configs.split(",")]
    Ps = [S.load_dtu_projections()[i] for i in range(a.cams)]
    scale = 1600.0 / a.cols
    refs = list(range(a.cams)) if a.preset == "dtu" else list(range(0, a.cams, 2))
    fPs = [Ps[r] for r in refs]
    kw = dict(cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
    out = {"workload": "%d DTU cameras at %dx%d, %d reference views, %d iterations in all" % (a.cams, a.cols, a.rows, len(refs), a.iterations),
           "gpu": gpu, "geo_iterations": a.geo_iterations, "device_sets": device_sets}

    def params(iterations):
        p = S.AlgorithmParameters(box_hsize=11, box_vsize=11, iterations=iterations, n_best=3, cost_comb=S.COMB_BEST_N, gamma=10.0)
        p.depthMin, p.depthMax = 300.0, 800.0
        return p

    def timed(fn):
        t0 = time.perf_counter()
        r = fn()
        return r, round(time.perf_counter() - t0, 3)

    def log(msg):
        print("geo_bench: %s" % msg, file=sys.stderr, flush=True)

    def per_iteration_ms(seconds, iterations):
        return round(1e3 * float(np.median(seconds)) / iterations, 3) if iterations else None

    for scene in a.scenes.split(","):
        log("%s: rendering %d views and the ground truth" % (scene, a.cams))
        cams = S.prepare_cameras(Ps, scale)
        hf = S.HeightField(z0=550.0, unit=550.0 / cams[0].fx, seed=77, hard=scene == "hard")
        images = np.stack([S.render_view(c, a.rows, a.cols, hf, noise_seed=(1000 + i) if hf.hard else None)[0]
                           for i, c in enumerate(cams)])
        gt = S.gt_points(fPs, scale, a.rows, a.cols, hf, stride=stride)
        unit = hf.unit
        taus = (0.25 * unit, 0.5 * unit, unit)

        def score(n4):
            v, _ = api.fuse(n4, fPs, cam_scale=scale, **fuse_kw)
            s = api.evaluate_cloud(v, gt, max_dist=10 * unit, taus=taus)
            return {"vertices": len(v), "accuracy_mean_units": round(s["accuracy_mean"] / unit, 4),
                    "completeness_mean_units": round(s["completeness_mean"] / unit, 4),
                    "f_score": [round(f, 4) for f in s["f_score"]]}

        res = {"unit": unit, "gt_points": len(gt)}
        first = {}
        for k, devices in enumerate(device_sets):
            name = ",".join(str(d) for d in devices)
            api.batch_run(images, Ps, params(1), refs[:1], devices=devices, want_outputs=False, **kw)      # warm-up
            runs = [("photometric", lambda: api.batch_run(images, Ps, params(a.iterations), refs, devices=devices, **kw))]
            runs += [("geometric w=%g max_err=%g" % (w, m),
                      lambda w=w, m=m: api.geometric_pass(images, Ps, params(a.iterations - a.geo_iterations), refs,
                                                          geo_iterations=a.geo_iterations, weight=w, max_err=m, devices=devices, **kw))
                     for w, m in configs]
            for key, run in runs:
                (n4, _, info), wall = timed(run)
                if k == 0:
                    res[key], first[key] = score(n4), n4
                else:
                    assert np.array_equal(n4.view(np.uint32), first[key].view(np.uint32)), "%s: devices %s differ" % (key, name)
                r = res[key]
                r.setdefault("wall_s", {})[name] = wall
                log("%s, %s, devices %s: %.3f s" % (scene, key, name, wall))
                if key != "photometric":
                    r["pass1_views"] = len(info["pass1_views"])
                    r.setdefault("pass1_ms_per_iteration", {})[name] = per_iteration_ms(info["pass1_sweep_s"], a.iterations - a.geo_iterations)
                    r.setdefault("pass2_ms_per_iteration", {})[name] = per_iteration_ms(info["pass2_sweep_s"], a.geo_iterations)
                del n4, info
        out[scene] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Fused-cloud quality, scale dependence and speed of the fusion's two consistency rules (DESIGN.md §22); prints one JSON line.

    python tools/fuse_rule_bench.py [--rows 600] [--cols 800] [--cams 16] [--scenes smooth,hard,lit] [--costs pm,ncc]
                                    [--no-dtu]

Quality: tools/ms_bench.py's workload (the first `--cams` DTU cameras at `--cols` x `--rows`, every second camera a
reference view, box 11, n_best 3, depth 300..800, views at 5..45 degrees, at most 6 per reference; scenes smooth, hard and
lit; PM and NCC).  Per scene and cost, three runs: batch_run 6, geometric_pass 4 + 2 and multiscale_pass at 2 levels with
the detail restorer at its defaults.  Each run's outputs are fused with the disparity rule (disp_thresh 0.1, 30 degrees,
num_consistent 2) and with the reprojection rule at FUSE_REPROJ_DEFAULTS x normal_thresh {30, 10} x num_consistent {2, 3};
each row has the F-score at 0.25, 0.5 and 1 unit, mean accuracy and completeness (units) and vertices, and on the hard
scene the F-score at 1 unit of the points within ms_bench.EDGE_UNITS units of a block wall.
Scale: the same outputs fused in the world scaled by 2^-10 (P's fourth column, the depths and the depth range times
2^-10) with each rule's thresholds of the first two rows, scored against the scaled ground truth at scaled distances.
Speed (unless --no-dtu): fuse_ms of both rules on 49 DTU cameras at 1600 x 1200 with ground-truth maps (num_consistent 3),
one warm-up call each, then 5 calls per rule alternating: median, min and max.
Needs a CUDA device; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

SCALE = 2.0 ** -10


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600)
    ap.add_argument("--cols", type=int, default=800)
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--scenes", default="smooth,hard,lit")
    ap.add_argument("--costs", default="pm,ncc")
    ap.add_argument("--no-dtu", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("fuse_rule_bench: needs a CUDA device")
    from gipuma_b200 import api, scene as S
    from ms_bench import EDGE_UNITS, near_wall
    gpu = {"name": torch.cuda.get_device_name(0)}
    try:
        gpu["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.split()
    except Exception as e:      # noqa: BLE001
        gpu["power_limit_w"] = "unknown (%s)" % e

    def log(msg):
        print("fuse_rule_bench: %s" % msg, file=sys.stderr, flush=True)

    base = dict(depth_min=300.0, depth_max=800.0)
    rules = {"disparity 0.1, 30 deg, 2": dict(disp_thresh=0.1, normal_thresh=30.0, num_consistent=2)}
    for nt in (30.0, 10.0):
        for nc in (2, 3):
            rules["reprojection %g px, %g, %g deg, %d" % (api.FUSE_REPROJ_DEFAULTS["reproj_px"], api.FUSE_REPROJ_DEFAULTS["depth_rel"],
                                                          nt, nc)] = dict(rule="reprojection", normal_thresh=nt, num_consistent=nc)
    scale_rows = list(rules)[:2]
    out = {"gpu": gpu, "workload": "%d DTU cameras at %dx%d" % (a.cams, a.cols, a.rows),
           "fuse_reproj_defaults": api.FUSE_REPROJ_DEFAULTS, "edge_units": EDGE_UNITS, "scale": SCALE}

    def params(iterations):
        p = S.AlgorithmParameters(box_hsize=11, box_vsize=11, iterations=iterations, n_best=3, cost_comb=S.COMB_BEST_N, gamma=10.0)
        p.depthMin, p.depthMax = 300.0, 800.0
        return p

    Ps = [S.load_dtu_projections()[i] for i in range(a.cams)]
    scale = 1600.0 / a.cols
    refs = list(range(0, a.cams, 2))
    fPs = [Ps[r] for r in refs]
    sPs = [np.hstack([np.asarray(P, np.float64)[:, :3], np.asarray(P, np.float64)[:, 3:] * SCALE]) for P in fPs]
    kw = dict(cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
    costs = {"pm": {}, "ncc": dict(photometric="ncc", ncc_min_std=api.NCC_MIN_STD)}
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

        def score(v, gt_pts, u):
            s = api.evaluate_cloud(v, gt_pts, max_dist=10 * u, taus=(0.25 * u, 0.5 * u, u))
            return {"f_score": [round(f, 4) for f in s["f_score"]], "accuracy_mean_units": round(s["accuracy_mean"] / u, 4),
                    "completeness_mean_units": round(s["completeness_mean"] / u, 4), "vertices": len(v)}

        def fused(n4):
            row = {}
            for name, r in rules.items():
                v, _ = api.fuse(n4, fPs, cam_scale=scale, **base, **r)
                row[name] = score(v, gt, unit)
                if scene == "hard":
                    p = np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float32)
                    ev, eg = near_wall(p[:, 0], p[:, 1], unit), near_wall(gt[:, 0], gt[:, 1], unit)
                    e = api.evaluate_cloud(np.ascontiguousarray(p[ev]), np.ascontiguousarray(gt[eg]), max_dist=10 * unit, taus=(unit,))
                    row[name]["edge_f_score_1unit"] = round(e["f_score"][0], 4)
            sn4 = n4.copy()
            sn4[..., 3] *= np.float32(SCALE)
            for name in scale_rows:
                v, _ = api.fuse(sn4, sPs, cam_scale=scale, depth_min=base["depth_min"] * SCALE,
                                depth_max=base["depth_max"] * SCALE, **rules[name])
                row[name]["scaled_world"] = score(v, np.ascontiguousarray(gt * np.float32(SCALE)), unit * SCALE)
            return row

        res = {}
        for cost, photo in costs.items():
            if cost not in a.costs.split(","):
                continue
            n4, _, _ = api.batch_run(images, Ps, params(6), refs, **kw, **photo)
            res["%s batch_run 6" % cost] = fused(n4)
            n4, _, _ = api.geometric_pass(images, Ps, params(4), refs, geo_iterations=2, **kw, **photo)
            res["%s geometric_pass 4 + 2" % cost] = fused(n4)
            n4, _, _ = api.multiscale_pass(images, Ps, params(4), refs, levels=2, geo_iterations=2, detail_restorer={}, **kw, **photo)
            res["%s multiscale_pass 2 levels, restorer" % cost] = fused(n4)
            for k in list(res)[-3:]:
                log("%s %s: %s" % (scene, k, res[k]))
        out[scene] = res

    if not a.no_dtu:
        Ps = [S.load_dtu_projections()[i] for i in range(49)]
        log("DTU size: rendering ground truth")
        hf = S.HeightField(z0=550.0, unit=550.0 / S.prepare_cameras(Ps[:1])[0].fx, seed=77)
        gt = torch.from_numpy(S.render_norm4(Ps, 1.0, 1200, 1600, hf)).cuda()     # device maps: fuse_ms alone is timed
        prm = dict(base, normal_thresh=30.0, num_consistent=3)
        speed = {"disparity": dict(disp_thresh=0.1), "reprojection": dict(rule="reprojection")}
        times = {k: [] for k in speed}
        counts = {}
        for k, r in speed.items():
            counts[k] = api.fuse(gt, Ps, **prm, **r)[1]["count"]                       # warm-up
        for _ in range(5):
            for k, r in speed.items():
                times[k].append(api.fuse(gt, Ps, **prm, **r)[1]["fuse_ms"])
        out["dtu_speed"] = {k: {"fuse_ms_median": round(float(np.median(t)), 2), "fuse_ms_min": round(min(t), 2),
                                "fuse_ms_max": round(max(t), 2), "vertices": counts[k]} for k, t in times.items()}
        out["dtu_speed"]["workload"] = "49 DTU cameras at 1600x1200, ground-truth maps on the device, num_consistent 3"
        log("DTU size: %s" % out["dtu_speed"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()

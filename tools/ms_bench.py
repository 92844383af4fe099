"""Fused-cloud quality and sweep time of coarse-to-fine multi-scale PatchMatch (DESIGN.md §19) against the single-scale flows;
prints one JSON line.

    python tools/ms_bench.py [--rows 600] [--cols 800] [--cams 16] [--scenes smooth,hard,lit] [--costs pm,ncc]
                             [--modes fixed,adaptive] [--levels 2,3] [--weights 0.5,0] [--jbu RADIUS,SIGMA_S,SIGMA_R] [--dtu-preset]
                             [--prior] [--restore]

Quality: tools/acs_bench.py's workload (the first `--cams` DTU cameras at `--cols` x `--rows`, every second camera a
reference view, box 11, n_best 3, depth 300..800, views at 5..45 degrees, at most 6 per reference; the same fusion and
evaluate_cloud set-up; scenes smooth, hard and lit).  Per scene, cost and propagation, the rows are batch_run with 6
iterations, geometric_pass with 4 + 2, and multiscale_pass with 4 photometric iterations at the coarsest level and 2 with the
geometric term at every level, at each of `--levels` and `--weights` (weight 0: coarse-to-fine without the term).  Each row
has the F-score at 0.25, 0.5 and 1 unit, mean accuracy and completeness (units), vertices and the sweep ms summed over every
level and view (CUDA events on gpm_stream); on the hard scene also the scores on its texture-less band (acs_bench.py's
prior_study band rule).  --dtu-preset adds 49 cameras at 1600 x 1200, every camera a reference view, PM, one worker:
wall seconds and summed sweep seconds of geometric_pass 4 + 2 against multiscale_pass at each of `--levels`.
--prior adds the planar prior inside the multi-level driver (DESIGN.md §20), each stage with PRIOR_DEFAULTS and 2 sweeps: per
level count, multiscale_pass at weight GEO_WEIGHT with no stage, the photometric stage, the geometric stage and both, the
geometric stage at two support costs (PRIOR_DEFAULTS["support_cost"] and that plus GEO_WEIGHT * 1 pixel, the geometric term
of a pixel 1 pixel off), with the prior builds' host ms per level; and geometric_pass 4 + 2 with planar_prior as the
single-scale comparison.  With --dtu-preset it adds multiscale_pass with both stages at each support cost to the preset.
--restore adds the detail restorer (DESIGN.md §21): per level count, multiscale_pass at weight GEO_WEIGHT without it and with
it at each threshold of RESTORE_THRESHOLDS for the cost (RESTORE_DEFAULTS otherwise), with the share of level-0 pixels
restored and the wall seconds of the call; on the hard scene every row also has the edge scores: F at 1 unit and mean
completeness of the points within EDGE_UNITS units of a block wall (HeightField.height's block rule).  With --dtu-preset it
adds multiscale_pass with the restorer at its defaults to the preset.
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

RESTORE_THRESHOLDS = {"pm": (0.5, 1.0, 2.0), "ncc": (0.05, 0.1, 0.2)}
EDGE_UNITS = 3.0


def near_wall(X, Y, unit, k=EDGE_UNITS):
    """Points within k units of a block wall of HeightField.height: blocks are u < 0.33 and w < 0.33 of a 520-unit lattice,
    u = X / 520 + 0.31, w = Y / 520 + 0.17 (mod 1)."""
    L = 520.0 * unit
    u, w = np.mod(X / L + 0.31, 1.0), np.mod(Y / L + 0.17, 1.0)
    ku = k * unit / L

    def dist(t):                                   # lattice distance to the nearest wall line, 0 or 0.33
        return np.minimum(np.minimum(t, 1.0 - t), np.abs(t - 0.33))
    inside = lambda t: (t < 0.33 + ku) | (t > 1.0 - ku)           # noqa: E731  (within the block's span, walls included)
    return ((dist(u) < ku) & inside(w)) | ((dist(w) < ku) & inside(u))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600)
    ap.add_argument("--cols", type=int, default=800)
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--scenes", default="smooth,hard,lit")
    ap.add_argument("--costs", default="pm,ncc")
    ap.add_argument("--modes", default="fixed,adaptive")
    ap.add_argument("--levels", default="2,3")
    ap.add_argument("--weights", default="0.5,0")
    ap.add_argument("--jbu", default="")
    ap.add_argument("--dtu-preset", action="store_true")
    ap.add_argument("--prior", action="store_true")
    ap.add_argument("--restore", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ms_bench: needs a CUDA device")
    from gipuma_b200 import api, scene as S
    gpu = {"name": torch.cuda.get_device_name(0)}
    try:
        gpu["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.split()
    except Exception as e:      # noqa: BLE001
        gpu["power_limit_w"] = "unknown (%s)" % e

    def log(msg):
        print("ms_bench: %s" % msg, file=sys.stderr, flush=True)

    jbu = dict(api.JBU_DEFAULTS)
    if a.jbu:
        r, ss, sr = a.jbu.split(",")
        jbu = {"radius": int(r), "sigma_space": float(ss), "sigma_range": float(sr)}
    levels = [int(x) for x in a.levels.split(",") if x]
    weights = [float(x) for x in a.weights.split(",") if x]
    out = {"gpu": gpu, "jbu": jbu, "workload": "%d DTU cameras at %dx%d" % (a.cams, a.cols, a.rows)}
    costs = {"pm": {}, "ncc": dict(photometric="ncc", ncc_min_std=api.NCC_MIN_STD)}
    costs = {k: costs[k] for k in a.costs.split(",") if k}
    s0 = api.PRIOR_DEFAULTS["support_cost"]
    supports = [s0, s0 + api.GEO_WEIGHT * 1.0]
    prior_rows = [("none", None, None), ("photometric", {}, None)]
    prior_rows += [(name % s, photo, {"support_cost": s}) for s in supports
                   for name, photo in (("geometric s=%g", None), ("both s=%g", {}))]
    if a.prior:
        out["prior_support_costs"] = supports

    def params(iterations):
        p = S.AlgorithmParameters(box_hsize=11, box_vsize=11, iterations=iterations, n_best=3, cost_comb=S.COMB_BEST_N, gamma=10.0)
        p.depthMin, p.depthMax = 300.0, 800.0
        return p

    def render(Ps, scale, rows, cols, hard):
        cams = S.prepare_cameras(Ps, scale)
        hf = S.HeightField(z0=550.0, unit=550.0 / cams[0].fx, seed=77, hard=hard)
        images = np.stack([S.render_view(c, rows, cols, hf, noise_seed=(1000 + i) if hf.hard else None)[0]
                           for i, c in enumerate(cams)]).astype(np.float32)
        return hf, images

    Ps = [S.load_dtu_projections()[i] for i in range(a.cams)]
    scale = 1600.0 / a.cols
    refs = list(range(0, a.cams, 2))
    fPs = [Ps[r] for r in refs]
    kw = dict(cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
    fuse_kw = dict(depth_min=300.0, depth_max=800.0, disp_thresh=0.1, normal_thresh=30.0, num_consistent=2)
    for scene in [x for x in a.scenes.split(",") if x]:
        log("%s: rendering" % scene)
        hf, images = render(Ps, scale, a.rows, a.cols, scene == "hard")
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
                ev, eg = near_wall(v[:, 0], v[:, 1], unit), near_wall(gt[:, 0], gt[:, 1], unit)
                e = api.evaluate_cloud(np.ascontiguousarray(v[ev]), np.ascontiguousarray(gt[eg]), max_dist=10 * unit, taus=(unit,))
                r["edge_f_score_1unit"] = round(e["f_score"][0], 4)
                r["edge_completeness_mean_units"] = round(e["completeness_mean"] / unit, 4)
            return r

        res = {}
        for cost, photo in costs.items():
            for mode in [m for m in a.modes.split(",") if m]:
                row = {}
                n4, _, st = api.batch_run(images, Ps, params(6), refs, propagation=mode, **kw, **photo)
                row["batch_run 6"] = score(n4, st["sweep_ms_total"])
                n4, _, info = api.geometric_pass(images, Ps, params(4), refs, geo_iterations=2, propagation=mode, **kw, **photo)
                row["geometric_pass 4 + 2"] = score(n4, 1e3 * (sum(info["pass1_sweep_s"]) + sum(info["pass2_sweep_s"])))
                for L in levels:
                    for w in weights:
                        n4, _, info = api.multiscale_pass(images, Ps, params(4), refs, levels=L, geo_iterations=2, weight=w,
                                                          jbu=jbu, propagation=mode, **kw, **photo)
                        key = "multiscale_pass levels %d, weight %g" % (L, w)
                        row[key] = dict(score(n4, 1e3 * sum(info["level_sweep_s"])), views=len(info["views"]),
                                        level_sweep_ms=[round(1e3 * t, 1) for t in info["level_sweep_s"]],
                                        level_upsample_ms=[round(1e3 * t, 1) for t in info["level_upsample_s"]])
                        log("%s %s %s %s: %s" % (scene, cost, mode, key, row[key]))
                if a.prior:
                    n4, _, info = api.geometric_pass(images, Ps, params(4), refs, geo_iterations=2, propagation=mode,
                                                     planar_prior={}, **kw, **photo)
                    row["geometric_pass 4 + 2, planar_prior"] = score(n4, 1e3 * (sum(info["pass1_sweep_s"]) + sum(info["pass2_sweep_s"])))
                    for L in levels:
                        for name, pp, gp in prior_rows:
                            n4, _, info = api.multiscale_pass(images, Ps, params(4), refs, levels=L, geo_iterations=2, jbu=jbu,
                                                              propagation=mode, planar_prior=pp, geo_prior=gp, **kw, **photo)
                            key = "multiscale_pass levels %d, prior %s" % (L, name)
                            row[key] = dict(score(n4, 1e3 * sum(info["level_sweep_s"])),
                                            level_sweep_ms=[round(1e3 * t, 1) for t in info["level_sweep_s"]],
                                            level_build_ms=[round(t, 1) for t in info["level_build_ms"]])
                            log("%s %s %s %s: %s" % (scene, cost, mode, key, row[key]))
                if a.restore:
                    for L in levels:
                        for t in (None,) + RESTORE_THRESHOLDS[cost]:
                            t0 = time.perf_counter()
                            n4, _, info = api.multiscale_pass(images, Ps, params(4), refs, levels=L, geo_iterations=2, jbu=jbu,
                                                              propagation=mode, detail_restorer=None if t is None else {"threshold": t},
                                                              **kw, **photo)
                            wall = time.perf_counter() - t0
                            key = "multiscale_pass levels %d, %s" % (L, "no restorer" if t is None else "restorer t=%g" % t)
                            row[key] = dict(score(n4, 1e3 * sum(info["level_sweep_s"])), wall_s=round(wall, 2),
                                            level_sweep_ms=[round(1e3 * x, 1) for x in info["level_sweep_s"]],
                                            restored_share=None if t is None else round(sum(info["restored"]) / (len(refs) * a.rows * a.cols), 4))
                            log("%s %s %s %s: %s" % (scene, cost, mode, key, row[key]))
                res["%s %s" % (cost, mode)] = row
                log("%s %s %s: %s" % (scene, cost, mode, row))
        out[scene] = res

    if a.dtu_preset:
        n = 49
        allP = S.load_dtu_projections()[:n]
        log("DTU preset: rendering %d views at 1600x1200" % n)
        hf, images = render(allP, 1.0, 1200, 1600, False)
        dkw = dict(cam_scale=1.0, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
        dtu = {}
        t0 = time.perf_counter()
        _, _, info = api.geometric_pass(images, allP, params(4), list(range(n)), geo_iterations=2, **dkw)
        dtu["geometric_pass 4 + 2"] = {"wall_s": round(time.perf_counter() - t0, 2),
                                       "sweep_s_total": round(sum(info["pass1_sweep_s"]) + sum(info["pass2_sweep_s"]), 3)}
        for L in levels:
            t0 = time.perf_counter()
            _, _, info = api.multiscale_pass(images, allP, params(4), list(range(n)), levels=L, geo_iterations=2, jbu=jbu, **dkw)
            dtu["multiscale_pass levels %d" % L] = {"wall_s": round(time.perf_counter() - t0, 2),
                                                   "sweep_s_total": round(sum(info["level_sweep_s"]), 3),
                                                   "level_sweep_s": [round(t, 3) for t in info["level_sweep_s"]],
                                                   "level_upsample_s": [round(t, 3) for t in info["level_upsample_s"]]}
            for name, pp, gp in (prior_rows[-1:-4:-2] if a.prior else []):                # both stages, each support cost
                t0 = time.perf_counter()
                _, _, info = api.multiscale_pass(images, allP, params(4), list(range(n)), levels=L, geo_iterations=2, jbu=jbu,
                                                 planar_prior=pp, geo_prior=gp, **dkw)
                dtu["multiscale_pass levels %d, prior %s" % (L, name)] = {
                    "wall_s": round(time.perf_counter() - t0, 2), "sweep_s_total": round(sum(info["level_sweep_s"]), 3),
                    "level_sweep_s": [round(t, 3) for t in info["level_sweep_s"]],
                    "level_build_s": [round(t / 1e3, 3) for t in info["level_build_ms"]]}
            if a.restore:
                t0 = time.perf_counter()
                _, _, info = api.multiscale_pass(images, allP, params(4), list(range(n)), levels=L, geo_iterations=2, jbu=jbu,
                                                 detail_restorer={}, **dkw)
                dtu["multiscale_pass levels %d, restorer" % L] = {
                    "wall_s": round(time.perf_counter() - t0, 2), "sweep_s_total": round(sum(info["level_sweep_s"]), 3),
                    "level_sweep_s": [round(t, 3) for t in info["level_sweep_s"]],
                    "restored_share": round(sum(info["restored"]) / (n * 1600 * 1200), 4)}
        out["dtu_preset"] = dict(dtu, workload="%d views at 1600x1200, PM, fixed, one worker, every view a reference" % n)
        log("DTU preset: %s" % dtu)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

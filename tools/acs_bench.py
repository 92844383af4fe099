"""Fused-cloud quality, convergence and sweep speed of adaptive checkerboard sampling (DESIGN.md §16) against the reference's
fixed neighbours, and of joint view selection (§17) against the combination rule; prints one JSON line.

    python tools/acs_bench.py [--rows 600] [--cols 800] [--cams 16] [--iterations 6] [--geo-iterations 2]
                              [--converge 2,3,4,6] [--scenes smooth,hard,lit] [--costs pm,ncc] [--speed-iterations 4]
                              [--vsel off,joint] [--dtu-preset]

Quality: tools/ncc_bench.py's workload (the first `--cams` DTU cameras at `--cols` x `--rows`, every second camera a reference
view, box 11, n_best 3, depth 300..800, views at 5..45 degrees, at most 6 per reference; the same fusion and evaluate_cloud
set-up; scenes smooth, hard and lit).  Per scene, cost (PM, NCC at api.NCC_MIN_STD) and propagation (fixed, adaptive):
photometric only (batch_run, `--iterations`), with the geometric pass (geometric_pass, `--iterations` - `--geo-iterations`
photometric then `--geo-iterations` geometric iterations), and the photometric F-scores after each of `--converge`
iterations.  Each run reports F-score at 0.25, 0.5 and 1 unit, mean accuracy and completeness (units), vertices and the batch
driver's summed sweep ms per iteration (CUDA events on gpm_stream).
Speed: sweep ms per iteration from CUDA events on gpm_stream around gpm_sweep(`--speed-iterations`) after gpm_init and a
one-iteration warm-up, fixed against adaptive, PM and NCC, at 1600 x 1200 and 800 x 600 (10 views, box 15), with
gpm_get_stats' hypotheses offered, skipped and (view, sample) pairs evaluated of the timed sweep.
--dtu-preset adds a DTU-size batch: 49 cameras at 1600 x 1200, every camera a reference view, PM, one worker, fixed against
adaptive, total sweep seconds.
--vsel: the view selections to run with the NCC cost ("off", "joint" at api.JVS_DEFAULTS; PM runs "off" only): every NCC
quality and speed row is repeated per view selection (keys "<cost> <propagation>" and "<cost> <propagation> joint"), and
--dtu-preset adds NCC fixed without and with joint view selection.  Needs a CUDA device; there is no CPU path.
--prior PM_WEIGHTS/NCC_WEIGHTS (e.g. 1,4,16/0.1,0.3,1): the planar-prior study (DESIGN.md §18) instead of the above.  On the
same quality workload, per scene, cost and propagation, `--iterations` photometric iterations (batch_run) against
`--iterations` - 2 photometric plus 2 with the prior (planar_prior: sigma_d = (800 - 300) / 64, sigma_n 5 degrees, step 5,
support_cost 0.5 for NCC and 3 for PM) at each weight; on the hard scene also the scores restricted to its texture-less band
(ground-truth points with |Y - 180 unit| < 70 unit, the height field's band rule, and the vertices in the same band).  Then
the build time of gpm_build_planar_prior and sweep ms per iteration without and with the prior, at 800 x 600 and
1600 x 1200 (10 views, box 15, CUDA events on gpm_stream).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MODES = ("fixed", "adaptive")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600)
    ap.add_argument("--cols", type=int, default=800)
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--iterations", type=int, default=6)
    ap.add_argument("--geo-iterations", type=int, default=2)
    ap.add_argument("--converge", default="2,3,4,6")
    ap.add_argument("--scenes", default="smooth,hard,lit")
    ap.add_argument("--costs", default="pm,ncc")
    ap.add_argument("--speed-iterations", type=int, default=4)
    ap.add_argument("--vsel", default="off")
    ap.add_argument("--dtu-preset", action="store_true")
    ap.add_argument("--prior", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("acs_bench: needs a CUDA device")
    from gipuma_b200 import api, scene as S
    gpu = {"name": torch.cuda.get_device_name(0)}
    try:
        gpu["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.split()
    except Exception as e:      # noqa: BLE001
        gpu["power_limit_w"] = "unknown (%s)" % e

    def log(msg):
        print("acs_bench: %s" % msg, file=sys.stderr, flush=True)

    out = {"gpu": gpu, "workload": "%d DTU cameras at %dx%d, %d iterations (geometric: last %d)" %
           (a.cams, a.cols, a.rows, a.iterations, a.geo_iterations)}
    converge = [int(x) for x in a.converge.split(",") if x]
    costs = {"pm": {}, "ncc": dict(photometric="ncc", ncc_min_std=api.NCC_MIN_STD)}
    costs = {k: costs[k] for k in a.costs.split(",") if k}
    vsels = [v for v in a.vsel.split(",") if v]

    def runs(cost):
        """(key, propagation, view selection) of one cost: joint view selection is built for NCC only"""
        return [("%s %s%s" % (cost, mode, "" if v == "off" else " " + v), mode, v) for mode in MODES
                for v in (vsels if cost == "ncc" else ["off"])]

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
    if a.prior:
        out["prior"] = prior_study(a, api, S, torch, costs, render, params, Ps, scale, refs, fPs, kw, fuse_kw, log)
        print(json.dumps(out))
        return
    for scene in [x for x in a.scenes.split(",") if x]:                    # --scenes "": speed only
        log("%s: rendering" % scene)
        hf, images = render(Ps, scale, a.rows, a.cols, scene == "hard")
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

        for cost, photo in costs.items():
            for key, mode, vsel in runs(cost):
                r = {}
                for it in sorted(set(converge + [a.iterations])):
                    n4, _, st = api.batch_run(images, Ps, params(it), refs, propagation=mode, view_selection=vsel, **kw, **photo)
                    sc = score(n4)
                    if it == a.iterations:
                        r["photometric"] = dict(sc, sweep_ms_per_iteration=round(st["sweep_ms_total"] / it, 2))
                    if it in converge:
                        r.setdefault("f_score_1unit_after_iterations", {})[it] = sc["f_score"][2]
                n4, _, info = api.geometric_pass(images, Ps, params(a.iterations - a.geo_iterations), refs,
                                                 geo_iterations=a.geo_iterations, propagation=mode, view_selection=vsel, **kw, **photo)
                r["with_geometric"] = dict(score(n4), pass2_sweep_ms_per_iteration=round(
                    1e3 * sum(info["pass2_sweep_s"]) / max(1, a.geo_iterations), 2))
                res[key] = r
                log("%s %s: %s" % (scene, key, r))
        out[scene] = res

    speed = {}
    for rows, cols in ((1200, 1600), (600, 800)):
        sc = S.make_config(2, rows=rows, cols=cols, n_views=10, iterations=1, seed=7)
        sc.params.box_hsize = sc.params.box_vsize = 15
        row = {}
        for cost in costs:
            for key, mode, vsel in runs(cost):
                with api.Context(cols, rows, len(sc.subset)) as ctx:
                    ctx.load_scene(sc)
                    if cost == "ncc":
                        ctx.set_photometric("ncc", api.NCC_MIN_STD)
                    ctx.set_propagation(mode)
                    ctx.set_view_selection(vsel)
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
                    row[key] = {"ms_per_iteration": round(e0.elapsed_time(e1) / a.speed_iterations, 3),
                                                   "offered": st["hypotheses"], "skipped": st["skipped"], "pairs": st["pairs"]}
            row["%s adaptive_over_fixed" % cost] = round(row["%s adaptive" % cost]["ms_per_iteration"] /
                                                         row["%s fixed" % cost]["ms_per_iteration"], 3)
            if cost == "ncc" and "joint" in vsels:
                for mode in MODES:
                    row["ncc %s joint_over_off" % mode] = round(row["ncc %s joint" % mode]["ms_per_iteration"] /
                                                                row["ncc %s" % mode]["ms_per_iteration"], 3)
        speed["%dx%d, 10 views, box 15" % (cols, rows)] = row
        log("speed %dx%d: %s" % (cols, rows, row))
    out["speed"] = speed

    if a.dtu_preset:
        n = 49
        allP = S.load_dtu_projections()[:n]
        log("DTU preset: rendering %d views at 1600x1200" % n)
        hf, images = render(allP, 1.0, 1200, 1600, False)
        dtu = {}
        for mode in MODES:
            t0 = time.perf_counter()
            _, _, st = api.batch_run(images, allP, params(a.iterations), list(range(n)), cam_scale=1.0, min_angle=5.0,
                                     max_angle=45.0, max_views=6, seed=4242, want_outputs=False, propagation=mode)
            dtu[mode] = {"sweep_s_total": round(st["sweep_ms_total"] / 1e3, 3), "wall_s": round(time.perf_counter() - t0, 2)}
        dtu["adaptive_over_fixed"] = round(dtu["adaptive"]["sweep_s_total"] / dtu["fixed"]["sweep_s_total"], 3)
        if "joint" in vsels:
            for vsel in ("off", "joint"):
                t0 = time.perf_counter()
                _, _, st = api.batch_run(images, allP, params(a.iterations), list(range(n)), cam_scale=1.0, min_angle=5.0,
                                         max_angle=45.0, max_views=6, seed=4242, want_outputs=False, photometric="ncc",
                                         ncc_min_std=api.NCC_MIN_STD, view_selection=vsel)
                dtu["ncc fixed " + vsel] = {"sweep_s_total": round(st["sweep_ms_total"] / 1e3, 3),
                                            "wall_s": round(time.perf_counter() - t0, 2)}
            dtu["ncc joint_over_off"] = round(dtu["ncc fixed joint"]["sweep_s_total"] / dtu["ncc fixed off"]["sweep_s_total"], 3)
        out["dtu_preset"] = dict(dtu, workload="%d views at 1600x1200, PM, %d iterations, one worker" % (n, a.iterations))
        log("DTU preset: %s" % dtu)
    print(json.dumps(out))


def prior_study(a, api, S, torch, costs, render, params, Ps, scale, refs, fPs, kw, fuse_kw, log):
    pm_w, ncc_w = a.prior.split("/")
    weights = {"pm": [float(x) for x in pm_w.split(",") if x], "ncc": [float(x) for x in ncc_w.split(",") if x]}
    support = {"pm": 3.0, "ncc": 0.5}
    sigma_d = (800.0 - 300.0) / 64.0
    res = {}
    for scene in [x for x in a.scenes.split(",") if x]:
        log("prior %s: rendering" % scene)
        hf, images = render(Ps, scale, a.rows, a.cols, scene == "hard")
        if scene == "lit":
            rng = np.random.default_rng(2024)
            images = np.clip(np.stack([rng.uniform(0.6, 1.4) * im + rng.uniform(-40, 40) for im in images]), 0, 255).astype(np.float32)
        gt = S.gt_points(fPs, scale, a.rows, a.cols, hf, stride=2)
        unit = hf.unit
        in_band = lambda p: np.abs(p[:, 1] - 180.0 * unit) < 70.0 * unit          # noqa: E731  (HeightField's band rule)

        def score(n4):
            v, _ = api.fuse(n4, fPs, cam_scale=scale, **fuse_kw)
            s = api.evaluate_cloud(v, gt, max_dist=10 * unit, taus=(0.25 * unit, 0.5 * unit, unit))
            r = {"f_score_1unit": round(s["f_score"][2], 4), "completeness_mean_units": round(s["completeness_mean"] / unit, 4)}
            if scene == "hard":
                v = np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float32)
                vb = np.ascontiguousarray(v[in_band(v)])
                b = api.evaluate_cloud(vb, np.ascontiguousarray(gt[in_band(gt)]), max_dist=10 * unit, taus=(unit,))
                r["band_f_score_1unit"] = round(b["f_score"][0], 4)
                r["band_completeness_mean_units"] = round(b["completeness_mean"] / unit, 4)
            return r

        row = {}
        for cost, photo in costs.items():
            for mode in MODES:
                key = "%s %s" % (cost, mode)
                n4, _, st = api.batch_run(images, Ps, params(a.iterations), refs, propagation=mode, **kw, **photo)
                r = {"photometric %d" % a.iterations: score(n4)}
                for w in weights[cost]:
                    prior = {"weight": w, "depth_sigma": sigma_d, "support_cost": support[cost], "iterations": 2}
                    n4, _, st = api.batch_run(images, Ps, params(a.iterations - 2), refs, propagation=mode, planar_prior=prior,
                                              **kw, **photo)
                    r["%d + 2 prior, weight %g" % (a.iterations - 2, w)] = dict(
                        score(n4), with_prior_share=round(float(np.mean([p["with_prior"] for p in st["prior"]])) / (a.rows * a.cols), 3))
                row[key] = r
                log("prior %s %s: %s" % (scene, key, r))
        res[scene] = row

    speed = {}
    for rows, cols in ((600, 800), (1200, 1600)):
        sc = S.make_config(2, rows=rows, cols=cols, n_views=10, iterations=1, seed=7)
        sc.params.box_hsize = sc.params.box_vsize = 15
        row = {}
        for cost in costs:
            with api.Context(cols, rows, len(sc.subset)) as ctx:
                ctx.load_scene(sc)
                if cost == "ncc":
                    ctx.set_photometric("ncc", api.NCC_MIN_STD)
                ctx.init()
                ctx.sweep(2)
                _, c = ctx.get_state()
                torch.cuda.synchronize()
                t = []
                for _ in range(3):
                    t0 = time.perf_counter()
                    info = ctx.build_planar_prior(5, float(np.nanpercentile(c, 50)))
                    t.append(time.perf_counter() - t0)
                stream = torch.cuda.ExternalStream(ctx.stream)
                r = {"build_ms": round(1e3 * min(t), 2), "build_counts": info}
                for label, w in (("without", 0.0), ("with", 1.0 if cost == "pm" else 0.3)):
                    ctx.set_prior(w, (sc.params.depthMax - sc.params.depthMin) / 64.0, 5.0)
                    p, _ = ctx.get_state()
                    ctx.set_state(p, ctx.cost_eval(p))
                    ctx.sweep(1)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    ctx.sweep(a.speed_iterations)
                    e1.record(stream)
                    e1.synchronize()
                    r["sweep_ms_per_iteration_%s_prior" % label] = round(e0.elapsed_time(e1) / a.speed_iterations, 3)
                row[cost] = r
        speed["%dx%d, 10 views, box 15" % (cols, rows)] = row
        log("prior speed %dx%d: %s" % (cols, rows, row))
    res["speed"] = speed
    return res


if __name__ == "__main__":
    main()

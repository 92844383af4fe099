"""Speed and surface quality of the meshing (gpm_tsdf_integrate + gpm_mesh_extract, DESIGN.md §24); prints one JSON line.

    python tools/mesh_bench.py [--rows 600] [--cols 800] [--cams 16] [--scenes smooth,hard,lit] [--costs pm,ncc]
                               [--flows batch,ms] [--refinements gipuma,acmh] [--voxels 0.5,1] [--truncs 2,3,5]
                               [--min-weights 1,2,3] [--no-dtu]

Speed (unless --no-dtu): 49 DTU cameras at 1600 x 1200, ground-truth maps (device inputs) into a 512^3 box around the
ground truth, trunc 3 voxels, min_weight 2: one warm-up, then 5 calls of each stage; median, min and max of integrate_ms and
extract_ms (CUDA events), the host-input upload_ms of one call, the vertex and face counts, the device bytes the two calls
allocate (computed from their buffers), and the single-thread C restatement's seconds on a slab of 4 z-slices of each stage.
Quality: ms_bench.py's workload (the first `--cams` DTU cameras at `--cols` x `--rows`, every second camera a reference
view, box 11, n_best 3, depth 300..800, views at 5..45 degrees, at most 6 per reference; scenes smooth, hard and lit).  Per
scene, cost (PM, NCC) and refinement (Gipuma's, ACMH's): batch_run with 6 iterations and multiscale_pass at 2 levels (4
photometric iterations, 2 with the geometric term).  Each run's depth maps are fused (reprojection rule, FUSE_REPROJ_DEFAULTS,
30 degrees, num_consistent 2) and meshed at every voxel (units) x trunc (voxels) x min_weight of the sweep, the mesh sampled
with sample_mesh at half a voxel.  Each row has F at 0.25, 0.5 and 1 unit, mean accuracy and completeness (units) and the
point / face counts, over the points in a cube of 192 units around the ground truth's median (the box the meshes are
made in, 3 voxels beyond it); on the hard scene also F at 1 unit and completeness on its texture-less band (ms_bench.py's rule).
`best` lists, per voxel, the (trunc, min_weight) of the highest mean F at 0.5 unit over every run.  The GPU's name and
power limit are read in the same run.  Needs a CUDA device; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

HALF = 96.0                 # half the side of the scored region, in units: 390 voxels per axis at half a unit


def _box(g, n, pad=3, voxel=None):
    lo, hi = g.min(axis=0).astype(np.float64), g.max(axis=0).astype(np.float64)
    if voxel is None:
        voxel = float(np.float32((hi - lo).max() / (n - 2 * pad)))
    origin = tuple(float(np.float32(x)) for x in lo - pad * voxel)
    dims = tuple(int(min(2048, np.ceil((hi[a] - lo[a]) / voxel) + 2 * pad)) for a in range(3))
    return origin, voxel, dims


def dtu_speed(api, S, log):
    import torch
    from oracle import pymesh
    Ps = [S.load_dtu_projections()[i] for i in range(49)]
    H, W = 1200, 1600
    hf = S.HeightField(z0=550.0, unit=550.0 / S.prepare_cameras(Ps[:1])[0].fx, seed=77)
    log("DTU: rendering ground truth")
    gt = S.render_norm4(Ps, 1.0, H, W, hf)
    dep = np.ascontiguousarray(gt[..., 3])
    origin, voxel, _ = _box(S.gt_points(Ps, 1.0, H, W, hf, stride=4, norm4=gt), 512)
    dims, trunc, mw = (512, 512, 512), 3.0 * voxel, 2
    dd = torch.from_numpy(dep).cuda()
    args = (origin, voxel, dims, trunc, 300.0, 800.0)
    D, Wt, _ = api.tsdf_integrate(dd, Ps, *args)
    v, f, _ = api.extract_mesh(D, Wt, origin, voxel, mw)
    ti, te = [], []
    for _ in range(5):
        D, Wt, i1 = api.tsdf_integrate(dd, Ps, *args)
        v, f, i2 = api.extract_mesh(D, Wt, origin, voxel, mw)
        ti.append(i1["integrate_ms"])
        te.append(i2["extract_ms"])
    _, _, ih = api.tsdf_integrate(dep, Ps, *args)
    nvox = 512 ** 3
    nblk = (nvox + 255) // 256
    out = {"workload": "49 DTU cameras at 1600x1200, ground-truth maps, 512^3 box, voxel %.4f, trunc 3 voxels, min_weight 2" % voxel,
           "integrate_ms": {"median": float(np.median(ti)), "min": min(ti), "max": max(ti)},
           "extract_ms": {"median": float(np.median(te)), "min": min(te), "max": max(te)},
           "upload_ms_host_inputs": ih["upload_ms"], "vertices": len(v), "faces": len(f),
           "device_bytes_integrate_host_inputs": dep.nbytes + 6 * nvox + 88 * 49,
           "device_bytes_extract": 6 * nvox + 2 * 4 * nblk + 2 * 8 * (nblk + 1) + 12 * len(v) + 12 * len(f)}
    Dh, Wh = D.cpu().numpy(), Wt.cpu().numpy()
    k0 = int(np.nonzero((Wh > 0).any(axis=(1, 2)))[0].mean())
    t0 = time.perf_counter()
    pymesh.tsdf(dep, api.fuse_cameras(Ps), origin, voxel, dims, trunc, 300.0, 800.0, (k0, k0 + 4), threads=1)
    t1 = time.perf_counter()
    pymesh.extract(Dh[k0:k0 + 4], Wh[k0:k0 + 4], origin, voxel, mw)
    t2 = time.perf_counter()
    out["restatement_single_thread_s_4_slices"] = {"integrate": round(t1 - t0, 3), "extract": round(t2 - t1, 3),
                                                   "gpu_ms_same_share": round(float(np.median(ti)) * 4 / 512, 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600)
    ap.add_argument("--cols", type=int, default=800)
    ap.add_argument("--cams", type=int, default=16)
    ap.add_argument("--scenes", default="smooth,hard,lit")
    ap.add_argument("--costs", default="pm,ncc")
    ap.add_argument("--flows", default="batch,ms")
    ap.add_argument("--refinements", default="gipuma,acmh")
    ap.add_argument("--voxels", default="0.5,1")
    ap.add_argument("--truncs", default="2,3,5")
    ap.add_argument("--min-weights", default="1,2,3")
    ap.add_argument("--no-dtu", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("mesh_bench: needs a CUDA device")
    from gipuma_b200 import api, scene as S
    gpu = {"name": torch.cuda.get_device_name(0)}
    try:
        gpu["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.split()
    except Exception as e:      # noqa: BLE001
        gpu["power_limit_w"] = "unknown (%s)" % e

    def log(msg):
        print("mesh_bench: %s" % msg, file=sys.stderr, flush=True)

    out = {"gpu": gpu}
    if not a.no_dtu:
        out["dtu"] = dtu_speed(api, S, log)
        log("DTU: %s" % out["dtu"])
    fl = lambda s, f=float: [f(x) for x in s.split(",") if x]           # noqa: E731
    voxels, truncs, mws = fl(a.voxels), fl(a.truncs), fl(a.min_weights, int)
    costs = {"pm": {}, "ncc": dict(photometric="ncc", ncc_min_std=api.NCC_MIN_STD)}
    refinements = {"gipuma": None, "acmh": {"kind": "acmh"}}

    def params(iterations):
        p = S.AlgorithmParameters(box_hsize=11, box_vsize=11, iterations=iterations, n_best=3, cost_comb=S.COMB_BEST_N, gamma=10.0)
        p.depthMin, p.depthMax = 300.0, 800.0
        return p

    Ps = [S.load_dtu_projections()[i] for i in range(a.cams)]
    scale = 1600.0 / a.cols
    refs = list(range(0, a.cams, 2))
    fPs = [Ps[r] for r in refs]
    kw = dict(cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
    fuse_kw = dict(depth_min=300.0, depth_max=800.0, normal_thresh=30.0, num_consistent=2, rule="reprojection")
    out["workload"] = "%d DTU cameras at %dx%d, %d reference views" % (a.cams, a.cols, a.rows, len(refs))
    sums = {}
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
        # the scored region: a cube of 2 * HALF units around the ground truth's median, clipped to its bounding box
        ctr = np.median(gt, axis=0).astype(np.float64)
        lo, hi = np.maximum(gt.min(axis=0), ctr - HALF * unit), np.minimum(gt.max(axis=0), ctr + HALF * unit)
        inside = lambda p: np.ascontiguousarray(p[((p >= lo) & (p <= hi)).all(axis=1)])      # noqa: E731
        gt = inside(gt)
        in_band = lambda p: np.abs(p[:, 1] - 180.0 * unit) < 70.0 * unit          # noqa: E731  (HeightField's band rule)

        def score(pts, extra):
            pts = inside(pts)
            s = api.evaluate_cloud(pts, gt, max_dist=10 * unit, taus=(0.25 * unit, 0.5 * unit, unit))
            r = {"f_score": [round(x, 4) for x in s["f_score"]], "accuracy_mean_units": round(s["accuracy_mean"] / unit, 4),
                 "completeness_mean_units": round(s["completeness_mean"] / unit, 4), "points": len(pts)}
            r.update(extra)
            if scene == "hard":
                b = api.evaluate_cloud(np.ascontiguousarray(pts[in_band(pts)]), np.ascontiguousarray(gt[in_band(gt)]),
                                       max_dist=10 * unit, taus=(unit,))
                r["band_f_score_1unit"] = round(b["f_score"][0], 4)
                r["band_completeness_mean_units"] = round(b["completeness_mean"] / unit, 4)
            return r

        res = {}
        for cost in [x for x in a.costs.split(",") if x]:
            for rname in [x for x in a.refinements.split(",") if x]:
                ref = refinements[rname]
                for flow in [x for x in a.flows.split(",") if x]:
                    if flow == "batch":
                        n4, _, _ = api.batch_run(images, Ps, params(6), refs, refinement=ref, **kw, **costs[cost])
                        name = "batch_run 6"
                    else:
                        n4, _, _ = api.multiscale_pass(images, Ps, params(4), refs, levels=2, geo_iterations=2, refinement=ref,
                                                       **kw, **costs[cost])
                        name = "multiscale_pass 2 levels"
                    key = "%s, %s, %s" % (name, cost, rname)
                    row = {}
                    v, _ = api.fuse(n4, fPs, cam_scale=scale, **fuse_kw)
                    fused = np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float32)
                    row["fused cloud"] = score(fused, {})
                    dep = np.ascontiguousarray(n4[..., 3])
                    for vox_units in voxels:
                        voxel = float(np.float32(vox_units * unit))
                        origin, voxel, dims = _box(np.stack([lo, hi]), 0, voxel=voxel)
                        for tv in truncs:
                            D, Wt, _ = api.tsdf_integrate(dep, fPs, origin, voxel, dims, tv * voxel, 300.0, 800.0, cam_scale=scale)
                            for mw in mws:
                                mv, mf, _ = api.extract_mesh(D, Wt, origin, voxel, mw)
                                pts = api.sample_mesh(mv, mf, voxel / 2) if len(mf) else np.zeros((0, 3), np.float32)
                                r = score(pts, {"faces": len(mf)})
                                row["mesh voxel %g, trunc %g, min_weight %d" % (vox_units, tv, mw)] = r
                                sums.setdefault((vox_units, tv, mw), []).append(r["f_score"][1])
                    log("%s %s: fused %s, mesh %s" % (scene, key, row["fused cloud"]["f_score"],
                                                      {k: r["f_score"] for k, r in row.items() if k.startswith("mesh voxel 1,")}))
                    res[key] = row
        out[scene] = res
    best = {}
    for vox in voxels:
        cand = {k: float(np.mean(x)) for k, x in sums.items() if k[0] == vox}
        if cand:
            k = max(cand, key=cand.get)
            best["voxel %g" % vox] = {"trunc_voxels": k[1], "min_weight": k[2], "mean_f_0.5unit": round(cand[k], 4),
                                      "all": {"trunc %g, min_weight %d" % (t, m): round(f, 4) for (_, t, m), f in cand.items()}}
    out["best"] = best
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""The planar prior inside the multi-level driver (ACMMP; DESIGN.md §20) on the GPU, every check bit for bit.

- gpm_ms_batch_run_prior with both stages NULL equals gpm_ms_batch_run and the restated multi-level flow of
  test_gpu_multiscale.py on every one of its cases;
- with the photometric stage, the geometric stage or both, it equals the multi-level flow restated here through Context
  calls (the prior stage: build_planar_prior, set_prior, set_state(cost_eval), offer_prior, sweep, and set_prior(0) after
  the keep or finalize), at two and three levels, PM fixed, NCC fixed and NCC adaptive, with 1, 2 and 3 workers on one GPU
  and over every GPU, in planes, costs and every info entry (per image index; zero where a view ran no stage);
- one level with the photometric stage only equals geometric_pass with planar_prior over V;
- a geometric stage that finds no support point equals its restatement and reports with_prior = 0 everywhere;
- the .dmb files equal the outputs, which fuse and score."""
import os

import numpy as np
import pytest

from conftest import bits_equal
from test_gpu_multiscale import CASES, GEO_ITERATIONS, JBU, KW, _closure, _device_lists, _restated, _run, _want

pytestmark = pytest.mark.gpu

DEPTH_SIGMA = (800.0 - 300.0) / 64                         # the test datasets' depth range over 64, as prior_opts derives it
MODES = {"pm_fixed": ("fusion", {}), "ncc_fixed": ("ragged", dict(photometric="ncc")),
         "ncc_adaptive": ("fusion", dict(photometric="ncc", propagation="adaptive"))}
STAGES = {"photometric": (True, False), "geometric": (False, True), "both": (True, True)}


def _prior(photometric, support_cost=1e30):
    return {"weight": 2.0 if photometric == "pm" else 0.1, "depth_sigma": DEPTH_SIGMA, "normal_sigma_deg": 5.0, "step": 5,
            "support_cost": support_cost, "iterations": 1}


def _restated_prior(images, Ps, params, refs, levels, cam_scale, min_angle, max_angle, max_views, seed, weight, max_err, jbu,
                    photo=None, geo=None, photometric="pm", propagation="fixed"):
    """test_gpu_multiscale._restated's flow with the two prior stages of §20.  Returns (norm4, cost, V, photometric counts
    {image: counts}, geometric counts {(level, image): counts})."""
    from gipuma_b200 import api
    import ctypes as C
    n, H, W = images.shape[:3]
    plan = _closure(Ps, refs, W, H, cam_scale, min_angle, max_angle, max_views)
    V = sorted(plan)
    size = [(api.level_size(W, l), api.level_size(H, l)) for l in range(levels)]
    pyr = {i: api.pyramid(images[i], levels) for i in V}

    def load(ctx, l, i):
        order, subset, (lo, hi) = plan[i]
        cams = api.prepare_cameras([Ps[k] for k in order], cam_scale * 2 ** l)
        ctx.set_photometric(photometric)
        ctx.set_propagation(propagation)
        ctx.set_view_selection("off")
        p = api.GpmParams.from_buffer_copy(api.pack_params(params))
        p.depthMin = p.depthMin if p.depthMin > 0 else lo
        p.depthMax = p.depthMax if p.depthMax > 0 else hi
        fb = np.float32(cams[0].f) * np.float32(cams[0].baseline)
        p.min_disparity, p.max_disparity = float(fb / np.float32(p.depthMax)), float(fb / np.float32(p.depthMin))
        ctx._check(ctx.lib.gpm_set_params(ctx.h, C.byref(p)))
        ctx.set_reference(pyr[i][l], cams[0])
        for v, k in enumerate(subset):
            ctx.set_view(v, pyr[order[k]][l], cams[k])
        ctx.set_num_views(len(subset))
        ctx.set_rng(seed, api.GPM_RNG_REFERENCE)
        return [order[k] for k in subset]

    def stage(ctx, P):
        counts = ctx.build_planar_prior(P["step"], P["support_cost"])
        ctx.set_prior(P["weight"], P["depth_sigma"], P["normal_sigma_deg"])
        planes, _ = ctx.get_state()
        ctx.set_state(planes, ctx.cost_eval(planes))
        ctx.offer_prior()
        ctx.sweep(P["iterations"])
        return counts

    def off(ctx, P):
        ctx.set_prior(0.0, P["depth_sigma"], P["normal_sigma_deg"])

    ctxs = [api.Context(w, h, max_views) for w, h in size]
    out, photo_counts, geo_counts = {}, {}, {}
    try:
        top = levels - 1
        raw, depth = {}, {}
        for i in V:
            c = ctxs[top]
            load(c, top, i)
            c.init()
            c.sweep(params.iterations)
            if photo:
                photo_counts[i] = stage(c, photo)
            raw[i] = c.get_state()[0]
            c.finalize()
            if photo:
                off(c, photo)
            depth[i] = np.ascontiguousarray(c.get_state()[0][..., 3])
        for l in range(top, -1, -1):
            ctx = ctxs[l]
            if l < top:
                up = {}
                for i in V:
                    load(ctx, l, i)
                    up[i] = ctx.upsample_planes(raw[i], **jbu)
                raw = {i: up[i][0] for i in V}
                depth = {i: up[i][1] for i in V}
            new_raw = {}
            for i in (V if l > 0 else sorted(set(refs))):
                src = load(ctx, l, i)
                for v, k in enumerate(src):
                    ctx.set_view_depth(v, depth[k])
                ctx.set_geometric(weight, max_err)
                ctx.set_state(raw[i], ctx.cost_eval(raw[i]))
                ctx.sweep(GEO_ITERATIONS)
                if geo:
                    geo_counts[(l, i)] = stage(ctx, geo)
                if l > 0:
                    new_raw[i] = ctx.get_state()[0]
                else:
                    ctx.finalize()
                    out[i] = ctx.get_state()
                if geo:
                    off(ctx, geo)
                ctx.set_geometric(0.0, max_err)
            raw = new_raw
    finally:
        for c in ctxs:
            c.close()
    n4 = np.stack([out[r][0] for r in refs])
    cc = np.stack([out[r][1] for r in refs])
    return n4, cc, V, photo_counts, geo_counts


_CACHE = {}


def _case_of(mode):
    from test_gpu_geometric_batch import _case
    name, modes = MODES[mode]
    c = _case(name, False)
    c["modes"] = modes
    return c


def _want_prior(mode, stages, levels, geo_support=1e30):
    from gipuma_b200 import api
    key = (mode, stages, levels, geo_support)
    if key not in _CACHE:
        c = _case_of(mode)
        photometric = c["modes"].get("photometric", "pm")
        on_photo, on_geo = STAGES[stages]
        photo = _prior(photometric) if on_photo else None
        geo = _prior(photometric, geo_support) if on_geo else None
        _CACHE[key] = (c, photo, geo, _restated_prior(c["images"], c["Ps"], c["params"], c["refs"], levels, c["scale"],
                                                      weight=api.GEO_WEIGHT, max_err=api.GEO_MAX_ERR, jbu=JBU, photo=photo,
                                                      geo=geo, **KW, **c["modes"]))
    return _CACHE[key]


def _check_info(info, n, levels, refs, V, photo, geo, photo_counts, geo_counts):
    zero = {"support": 0, "triangles": 0, "with_prior": 0}
    if photo:
        assert info["prior"]["photometric"] == [photo_counts.get(i, zero) for i in range(n)]
    else:
        assert info["prior"]["photometric"] is None
    if geo:
        assert info["prior"]["geometric"] == [[geo_counts.get((l, i), zero) for i in range(n)] for l in range(levels)]
        assert {(l, i) for (l, i) in geo_counts} == {(l, i) for l in range(levels) for i in (V if l else set(refs))}
    else:
        assert info["prior"]["geometric"] is None
    built = [bool(geo) or (bool(photo) and l == levels - 1) for l in range(levels)]
    assert [t > 0 for t in info["level_build_ms"]] == built


@pytest.mark.parametrize("levels", [2, 3])
@pytest.mark.parametrize("case", sorted(CASES))
def test_no_stage_equals_gpm_ms_batch_run(case, levels, monkeypatch):
    """multiscale_pass calls gpm_ms_batch_run_prior with both stages NULL; routed to gpm_ms_batch_run instead, it gives the
    same bits, and both equal test_gpu_multiscale's restated flow."""
    from gipuma_b200 import api
    c, (w4, wc, wV) = _want(case, levels)
    a4, ac, ainfo = _run(c, levels, devices=(0, 0))
    assert ainfo["prior"] == {"photometric": None, "geometric": None} and ainfo["level_build_ms"] == [0.0] * levels
    lib = api.load_library()
    plain = lib.gpm_ms_batch_run
    monkeypatch.setattr(lib, "gpm_ms_batch_run_prior", lambda m, o, v, po, st: plain(m, o, v, st))
    b4, bc, binfo = _run(c, levels, devices=(0, 0))
    assert bits_equal(a4, w4) == 0 and bits_equal(ac, wc) == 0
    assert bits_equal(b4, w4) == 0 and bits_equal(bc, wc) == 0
    assert ainfo["views"] == binfo["views"] == wV


@pytest.mark.parametrize("levels", [2, 3])
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("stages", sorted(STAGES))
def test_driver_equals_the_restated_flow_with_the_prior(stages, mode, levels):
    c, photo, geo, (w4, wc, wV, wp, wg) = _want_prior(mode, stages, levels)
    n = len(c["Ps"])
    assert all(k["with_prior"] > 0 for k in list(wp.values()) + list(wg.values()))
    for devices in _device_lists():
        n4, cost, info = _run(c, levels, devices=devices, planar_prior=photo, geo_prior=geo)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (stages, mode, levels, devices)
        assert info["views"] == wV, devices
        _check_info(info, n, levels, c["refs"], wV, photo, geo, wp, wg)
        assert len(info["level_sweep_s"]) == levels and all(t > 0 for t in info["level_sweep_s"])
    if stages == "both":                                   # each stage reaches the result
        for one in ("photometric", "geometric"):
            _, _, _, (o4, _, _, _, _) = _want_prior(mode, one, levels)
            assert bits_equal(o4, w4) > 0, one


def test_one_level_with_the_photometric_stage_is_geometric_pass_with_the_prior_over_the_view_set():
    from gipuma_b200 import api
    c = _case_of("ncc_fixed")
    photo = _prior("ncc")
    n4, cost, info = _run(c, 1, devices=(0, 0), planar_prior=photo)
    V = info["views"]
    g4, gc, ginfo = api.geometric_pass(c["images"], c["Ps"], c["params"], V, geo_iterations=GEO_ITERATIONS, cam_scale=c["scale"],
                                       devices=(0, 0), planar_prior=photo, **KW, **c["modes"])
    assert ginfo["pass1_views"] == V
    rows = [V.index(r) for r in c["refs"]]
    assert bits_equal(n4, g4[rows]) == 0 and bits_equal(cost, gc[rows]) == 0
    assert [info["prior"]["photometric"][i] for i in V] == ginfo["prior"]
    assert all(k["with_prior"] > 0 for k in ginfo["prior"])


@pytest.mark.parametrize("stages", ["geometric", "both"])
def test_a_geometric_stage_without_support_points_equals_its_restatement(stages):
    c, photo, geo, (w4, wc, wV, wp, wg) = _want_prior("pm_fixed", stages, 2, geo_support=-1.0)
    assert wg and all(k == {"support": 0, "triangles": 0, "with_prior": 0} for k in wg.values())
    n4, cost, info = _run(c, 2, devices=(0, 0, 0), planar_prior=photo, geo_prior=geo)
    assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0
    _check_info(info, len(c["Ps"]), 2, c["refs"], wV, photo, geo, wp, wg)
    assert all(k["with_prior"] == 0 for level in info["prior"]["geometric"] for k in level)


def test_dmb_files_equal_the_outputs_and_fuse_and_score(tmp_path):
    from gipuma_b200 import api
    from test_gpu_fusion import FUSE
    c, photo, geo, (w4, _, _, _, _) = _want_prior("pm_fixed", "both", 3)
    refs, Ps = c["refs"], c["Ps"]
    n4, _, _ = _run(c, 3, devices=(0, 0), out_dir=str(tmp_path), planar_prior=photo, geo_prior=geo)
    assert bits_equal(n4, w4) == 0
    for j, ref in enumerate(refs):
        d = api.read_dmb(os.path.join(str(tmp_path), "%08d" % ref, "disp.dmb"))
        nm = api.read_dmb(os.path.join(str(tmp_path), "%08d" % ref, "normals.dmb"))
        assert bits_equal(d, n4[j][..., 3]) == 0 and bits_equal(nm, n4[j][..., :3]) == 0
    v_mem, _ = api.fuse(n4, [Ps[r] for r in refs], cam_scale=c["scale"], **FUSE)
    v_dir, _ = api.fuse_batch_dir(str(tmp_path), refs, Ps, cam_scale=c["scale"], **FUSE)
    assert len(v_mem) > 1000 and v_mem.tobytes() == v_dir.tobytes()
    pts = np.stack([v_mem["x"], v_mem["y"], v_mem["z"]], 1)
    scores = api.evaluate_cloud(v_mem, pts[::3].copy(), max_dist=20.0)
    assert scores["n_rec"] == len(v_mem) and scores["f_score"][0] > 0

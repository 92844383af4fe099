"""The geometric term's per-pixel mask and the detail restorer (DESIGN.md §21) on the GPU, every check bit for bit.

- gpm_cost_eval with a random mask equals the per-pixel select (oracle/pyrestore.masked_cost) of the evaluations with the
  term on and off; an all-zero mask equals the term on, an all-ones mask the term off: PM and NCC, grey and colour, joint
  view selection, 4, 33 and 64 views;
- after init and sweeps, an all-zero mask equals the term on and an all-ones mask the term off, in planes and costs;
- with a random mask every propagation decision of every launch equals oracle/pypropagate.expected() with the masked cost,
  refinement keeps its invariants, and twins without memo, lower-bound early-out and duplicate skips, with one mask-7
  launch per colour, or at another warp count, stay bit-identical (windows 3, 15 and 25);
- setting and clearing the mask leaves the state alone and makes stored costs and the memo stale (while the term is on
  only); refusals change nothing;
- gpm_ms_batch_run_restore equals the flow restated here through Context calls, with and without a geometric prior stage,
  at two and three levels, PM fixed, NCC fixed and NCC adaptive with joint view selection, with 1-3 workers and over every
  GPU, in planes, costs, restored counts and every info entry;
- restore NULL equals gpm_ms_batch_run_prior;
- degenerate thresholds: none restored and no sweep gives the restorer-free planes; all restored and no sweep gives
  batch_run's planes with params.iterations = photo_iterations;
- the .dmb files equal the outputs, which fuse and score."""
import ctypes as C
import os
import time

import numpy as np
import pytest

from conftest import bits_equal
from test_gpu_geometric import MAX_ERR, WEIGHT, depth_maps, make_scene, open_ctx
from test_gpu_multiscale import GEO_ITERATIONS, JBU, KW, _closure, _device_lists, _run
from test_gpu_multiscale_prior import DEPTH_SIGMA, MODES, _case_of, _prior, _want_prior
from test_gpu_sweep_any_size import check_launch, cost_of

pytestmark = pytest.mark.gpu

f32 = np.float32
E_ARG = -1


def random_mask(sc, seed, share=0.5):
    return (np.random.default_rng(seed).random((sc.rows, sc.cols)) < share).astype(np.uint8)


def _modes(ctx, photometric, jvs):
    if photometric == "ncc":
        ctx.set_photometric("ncc")
    if jvs:
        ctx.set_view_selection("joint")


# rows, cols, views, colour, photometric, joint view selection
COSTS = [(53, 75, 4, False, "pm", False), (29, 41, 4, True, "pm", False), (53, 75, 4, False, "ncc", False),
         (53, 75, 4, False, "ncc", True), (40, 60, 33, False, "pm", False), (40, 60, 33, True, "pm", False),
         (40, 60, 33, False, "ncc", True), (40, 60, 64, False, "pm", False), (40, 60, 64, False, "ncc", False),
         (40, 60, 64, True, "pm", False)]


@pytest.mark.parametrize("rows,cols,views,color,photometric,jvs", COSTS)
def test_masked_cost_is_the_per_pixel_select(rows, cols, views, color, photometric, jvs):
    from oracle import pyrestore
    sc = make_scene(rows, cols, views, color=color)
    depths = depth_maps(sc, rows + views)
    mask = random_mask(sc, rows * cols + views)
    with open_ctx(sc, 5, depths, 0.0) as ctx:
        _modes(ctx, photometric, jvs)
        ctx.init()
        ctx.sweep(1)
        planes = [ctx.get_state()[0], np.random.default_rng(3).permutation(ctx.get_state()[0].reshape(-1, 4)).reshape(rows, cols, 4)]
        for p in planes:
            off = ctx.cost_eval(p)
            ctx.set_geo_mask(mask)                       # the term off: the mask has no effect
            assert bits_equal(ctx.cost_eval(p), off) == 0
            ctx.set_geometric(WEIGHT, MAX_ERR)
            masked = ctx.cost_eval(p)
            ctx.set_geo_mask(None)
            on = ctx.cost_eval(p)
            assert bits_equal(masked, pyrestore.masked_cost(on, off, mask)) == 0
            assert bits_equal(on, off) > 0               # the term changes costs, on both sides of the mask
            assert bits_equal(on[mask == 0], off[mask == 0]) > 0 and bits_equal(on[mask == 1], off[mask == 1]) > 0
            ctx.set_geo_mask(np.zeros_like(mask))
            assert bits_equal(ctx.cost_eval(p), on) == 0
            ctx.set_geo_mask(np.full_like(mask, 3))
            assert bits_equal(ctx.cost_eval(p), off) == 0
            ctx.set_geo_mask(None)
            ctx.set_geometric(0.0, MAX_ERR)


@pytest.mark.parametrize("rows,cols,views,color,photometric,jvs,adaptive",
                         [(53, 75, 4, False, "pm", False, False), (29, 41, 4, True, "pm", False, True),
                          (53, 75, 4, False, "ncc", True, True), (40, 60, 33, False, "ncc", False, False),
                          (40, 60, 64, False, "pm", False, True)])
def test_uniform_masks_sweep_as_the_term_on_and_off(rows, cols, views, color, photometric, jvs, adaptive):
    sc = make_scene(rows, cols, views, color=color)
    depths = depth_maps(sc, 11)
    outs = []
    for weight, mask in ((WEIGHT, None), (WEIGHT, 0), (0.0, None), (WEIGHT, 1)):
        with open_ctx(sc, 21, depths, weight) as ctx:
            _modes(ctx, photometric, jvs)
            if adaptive:
                ctx.set_propagation("adaptive")
            if mask is not None:
                ctx.set_geo_mask(np.full((rows, cols), mask, np.uint8))
            ctx.init()
            ctx.sweep(2)
            outs.append(ctx.get_state())
    for a, b in ((0, 1), (2, 3)):
        assert bits_equal(outs[a][0], outs[b][0]) == 0 and bits_equal(outs[a][1], outs[b][1]) == 0, (a, b)
    assert bits_equal(outs[0][0], outs[2][0]) > 0


# box 15: two rounds, so the lower bound is tested; box 25: six rounds; box 3: one round
@pytest.mark.parametrize("rows,cols,views,box,color", [(53, 75, 4, 15, False), (53, 75, 4, 15, True), (40, 60, 33, 3, False),
                                                       (40, 60, 33, 25, False), (40, 60, 64, 25, True)])
def test_masked_sweep_decisions_exact(rows, cols, views, box, color):
    from oracle import pypropagate as pp
    from oracle import pyrestore
    t0 = time.perf_counter()
    sc = make_scene(rows, cols, views, box=box, color=color)
    depths = depth_maps(sc, 3)
    mask = random_mask(sc, rows + box)
    seed = 4000 + rows + cols
    ctxs = [open_ctx(sc, seed, depths, WEIGHT),
            open_ctx(sc, seed, depths, WEIGHT, options={"memo": 0, "prune": 0, "dedupe": 0}),
            open_ctx(sc, seed, depths, WEIGHT),
            open_ctx(sc, seed, depths, WEIGHT, options={"nwarps": 3 if views == 64 else 7})]
    on, off = open_ctx(sc, seed, depths, WEIGHT), open_ctx(sc, seed, depths, 0.0)
    for ctx in ctxs:
        ctx.set_geo_mask(mask)
    A = ctxs[0]
    stepped = ctxs[1:2] + ctxs[3:]
    f_on, f_off = cost_of(on), cost_of(off)

    def f(planes, site):
        return pyrestore.masked_cost(f_on(planes, site), f_off(planes, site), mask)
    cam = sc.cameras[0]
    ys, xs = np.mgrid[0:sc.rows, 0:sc.cols]
    stats = {"compared": 0, "ambiguous": 0, "accepted": 0, "refined": 0}
    try:
        for ctx in ctxs:
            ctx.init()
        n0, c0 = A.get_state()
        for ctx in ctxs[1:]:
            assert bits_equal(ctx.get_state()[0], n0) == 0 and bits_equal(ctx.get_state()[1], c0) == 0
        A.reset_stats()
        for _ in range(2):
            for colour in (0, 1):
                for phase in (1, 2, 4):
                    before = A.get_state()
                    if phase != 4:
                        want_p, want_c, amb = pp.expected(before[0], before[1], colour, phase, f, cam, sc.params.depthMin,
                                                          sc.params.depthMax, color_images=color)
                    A.phase(colour, phase)
                    after = A.get_state()
                    for other in stepped:
                        other.phase(colour, phase)
                    p, c = ctxs[3].get_state()
                    assert bits_equal(p, after[0]) == 0 and bits_equal(c, after[1]) == 0, ("nwarps", colour, phase)
                    if phase != 4:
                        bad = ((after[0].view(np.uint32) != want_p.view(np.uint32)).any(axis=-1) |
                               (after[1].view(np.uint32) != want_c.view(np.uint32))) & ~amb
                        assert not bad.any(), (colour, phase, int(bad.sum()), np.argwhere(bad)[:8].tolist())
                        mine = ((xs + ys) & 1) == colour
                        stats["compared"] += int((mine & ~amb).sum())
                        stats["ambiguous"] += int((mine & amb).sum())
                        stats["accepted"] += int((mine & (after[1] < before[1])).sum())
                        check_launch(before, after, colour)
                    else:
                        stats["refined"] += check_launch(before, after, colour, f, sc, pp.refine_site(False, color))
                ctxs[2].phase(colour, 7)
                ref_p, ref_c = A.get_state()
                for other in ctxs[1:]:
                    p, c = other.get_state()
                    assert bits_equal(p, ref_p) == 0 and bits_equal(c, ref_c) == 0, colour
        st = A.stats()
    finally:
        for ctx in ctxs + [on, off]:
            ctx.close()
    share = stats["ambiguous"] / max(1, stats["compared"] + stats["ambiguous"])
    print("\nmasked geometric %dx%d, %d views, box %d, colour=%s: %s, ambiguous %.4f, pruned %d of %d, %.2f s" %
          (rows, cols, views, box, color, stats, share, st["pruned"], st["hypotheses"], time.perf_counter() - t0))
    assert stats["accepted"] > 0 and stats["refined"] > 0 and share <= 0.005
    if ((box - 1) // 2 + 1) ** 2 > 32:
        assert st["pruned"] > 0


def test_setting_and_clearing_the_mask_makes_costs_stale_and_leaves_the_state():
    sc = make_scene(53, 75, 4)
    depths = depth_maps(sc, 2)
    mask = random_mask(sc, 9)
    for weight in (WEIGHT, 0.0):
        ctxs = [open_ctx(sc, 77, depths, weight) for _ in range(2)]
        try:
            for ctx in ctxs:
                ctx.init()
                ctx.sweep(1)
            before = ctxs[0].get_state()
            ctxs[0].set_geo_mask(mask)
            mid = ctxs[0].get_state()
            ctxs[0].set_geo_mask(None)
            assert bits_equal(mid[0], before[0]) == 0 and bits_equal(mid[1], before[1]) == 0
            for ctx in ctxs:
                ctx.reset_stats()
                ctx.sweep(1)
            a, b = ctxs[0].get_state(), ctxs[1].get_state()
            assert bits_equal(a[0], b[0]) == 0 and bits_equal(a[1], b[1]) == 0
            ha, hb = ctxs[0].stats()["hypotheses"], ctxs[1].stats()["hypotheses"]
            if weight > 0:
                assert ha > hb, (ha, hb)                 # the memo was cleared and the costs' provenance forgotten
            else:
                assert ha == hb, (ha, hb)                # the term off: the mask changed nothing
        finally:
            for ctx in ctxs:
                ctx.close()


def test_refusals_change_nothing():
    from oracle import pyrestore
    sc = make_scene(31, 33, 4)
    depths = depth_maps(sc, 4)
    mask = random_mask(sc, 5)
    with open_ctx(sc, 3, depths, WEIGHT) as ctx, open_ctx(sc, 3, depths, WEIGHT) as on, open_ctx(sc, 3, depths, 0.0) as off:
        ctx.init()
        planes = ctx.get_state()[0]
        want = pyrestore.masked_cost(on.cost_eval(planes), off.cost_eval(planes), mask)
        ctx.set_geo_mask(mask)
        state = ctx.get_state()
        launches = ctx.stats()["launches"]
        bad = np.ascontiguousarray(np.ones((sc.rows, sc.cols), np.uint8))
        assert ctx.lib.gpm_set_geo_mask(ctx.h, C.c_void_p(bad.ctypes.data), sc.cols - 1, 0) == E_ARG
        assert "pitch" in ctx.lib.gpm_last_error().decode()
        ctx.set_planar_prior(np.zeros((sc.rows, sc.cols, 4), np.float32))
        with pytest.raises(Exception, match="mask and the planar prior"):
            ctx.set_prior(1.0, DEPTH_SIGMA)
        assert ctx.stats()["launches"] == launches
        s = ctx.get_state()
        assert bits_equal(s[0], state[0]) == 0 and bits_equal(s[1], state[1]) == 0
        assert bits_equal(ctx.cost_eval(planes), want) == 0              # the mask is still the one set
        ctx.set_geo_mask(None)
        ctx.set_prior(1.0, DEPTH_SIGMA)
        with pytest.raises(Exception, match="mask and the planar prior"):
            ctx.set_geo_mask(mask)
        ctx.set_prior(0.0, DEPTH_SIGMA)
        assert bits_equal(ctx.cost_eval(planes), on.cost_eval(planes)) == 0   # still no mask
        with pytest.raises(Exception, match="planar prior"):             # also while the term is off
            ctx.set_geometric(0.0, MAX_ERR)
            ctx.set_prior(1.0, DEPTH_SIGMA)
            ctx.set_geo_mask(mask)


# ---- the driver ----------------------------------------------------------------------------------------------------------

RESTORE = {"photo_iterations": 2, "threshold": 0.0, "iterations": 1}
DRIVER_MODES = {"pm_fixed": ("fusion", {}), "ncc_fixed": ("ragged", dict(photometric="ncc")),
                "ncc_adaptive_jvs": ("fusion", dict(photometric="ncc", propagation="adaptive", view_selection="joint"))}


def _restated_restore(images, Ps, params, refs, levels, cam_scale, min_angle, max_angle, max_views, seed, weight, max_err, jbu,
                      restore, geo=None, photometric="pm", propagation="fixed", view_selection="off"):
    """test_gpu_multiscale_prior's restated flow (no photometric stage) with the detail restorer at level 0.  Returns
    (norm4, cost, V, restored {ref: count})."""
    from gipuma_b200 import api
    from oracle import pyrestore
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
        ctx.set_view_selection(view_selection)
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
        ctx.build_planar_prior(P["step"], P["support_cost"])
        ctx.set_prior(P["weight"], P["depth_sigma"], P["normal_sigma_deg"])
        planes, _ = ctx.get_state()
        ctx.set_state(planes, ctx.cost_eval(planes))
        ctx.offer_prior()
        ctx.sweep(P["iterations"])

    ctxs = [api.Context(w, h, max_views) for w, h in size]
    out, restored = {}, {}
    try:
        top = levels - 1
        raw, depth = {}, {}
        for i in V:
            c = ctxs[top]
            load(c, top, i)
            c.init()
            c.sweep(params.iterations)
            raw[i] = c.get_state()[0]
            c.finalize()
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
                if l == 0:                                   # 1. the photometric-only estimate
                    load(ctx, 0, i)
                    ctx.init()
                    ctx.sweep(restore["photo_iterations"])
                    ph = ctx.get_state()[0]
                src = load(ctx, l, i)
                for v, k in enumerate(src):
                    ctx.set_view_depth(v, depth[k])
                ctx.set_geometric(weight, max_err)
                ctx.set_state(raw[i], ctx.cost_eval(raw[i]))
                ctx.sweep(GEO_ITERATIONS)
                if geo:
                    stage(ctx, geo)
                if l > 0:
                    new_raw[i] = ctx.get_state()[0]
                    if geo:
                        ctx.set_prior(0.0, geo["depth_sigma"], geo["normal_sigma_deg"])
                    ctx.set_geometric(0.0, max_err)
                    continue
                if geo:                                      # 2. the prior off, the geometric stage's planes
                    ctx.set_prior(0.0, geo["depth_sigma"], geo["normal_sigma_deg"])
                ms = ctx.get_state()[0]
                ctx.set_geometric(0.0, max_err)              # 3. detection
                detail = pyrestore.detect(ctx.cost_eval(ms), ctx.cost_eval(ph), restore["threshold"])
                merged = pyrestore.merge(ms, ph, detail)     # 4. restore
                ctx.set_geo_mask(detail)
                ctx.set_geometric(weight, max_err)
                ctx.set_state(merged, ctx.cost_eval(merged))
                ctx.sweep(restore["iterations"])
                ctx.finalize()                               # 5.
                out[i] = ctx.get_state()
                restored[i] = int(detail.sum())
                ctx.set_geo_mask(None)
                ctx.set_geometric(0.0, max_err)
            raw = new_raw
    finally:
        for c in ctxs:
            c.close()
    n4 = np.stack([out[r][0] for r in refs])
    cc = np.stack([out[r][1] for r in refs])
    return n4, cc, V, restored


_CACHE = {}


def _driver_case(mode):
    from test_gpu_geometric_batch import _case
    name, modes = DRIVER_MODES[mode]
    c = _case(name, False)
    c["modes"] = modes
    return c


def _want_restore(mode, levels, with_geo, restore=None):
    from gipuma_b200 import api
    restore = restore or RESTORE
    key = (mode, levels, with_geo, tuple(sorted(restore.items())))
    if key not in _CACHE:
        c = _driver_case(mode)
        geo = _prior(c["modes"].get("photometric", "pm"), 1.0) if with_geo else None
        _CACHE[key] = (c, geo, _restated_restore(c["images"], c["Ps"], c["params"], c["refs"], levels, c["scale"],
                                                 weight=api.GEO_WEIGHT, max_err=api.GEO_MAX_ERR, jbu=JBU, restore=restore, geo=geo,
                                                 **KW, **c["modes"]))
    return _CACHE[key]


@pytest.mark.parametrize("levels", [2, 3])
@pytest.mark.parametrize("mode,with_geo", [("pm_fixed", False), ("pm_fixed", True), ("ncc_fixed", False), ("ncc_fixed", True),
                                           ("ncc_adaptive_jvs", False)])
def test_driver_equals_the_restated_flow_with_the_restorer(mode, with_geo, levels):
    c, geo, (w4, wc, wV, wr) = _want_restore(mode, levels, with_geo)
    npix = c["images"].shape[1] * c["images"].shape[2]
    counts = [wr[r] for r in c["refs"]]
    assert all(0 < k < npix for k in counts), counts          # the restorer restored some pixels and kept others
    for devices in _device_lists():
        n4, cost, info = _run(c, levels, devices=devices, geo_prior=geo, detail_restorer=RESTORE)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (mode, with_geo, levels, devices)
        assert info["views"] == wV and info["restored"] == counts, devices
        assert len(info["level_sweep_s"]) == levels and all(t > 0 for t in info["level_sweep_s"])
        assert all(t > 0 for t in info["sweep_s"]) and all(d in devices for d in info["device"])
        assert (info["prior"]["geometric"] is not None) == with_geo and info["prior"]["photometric"] is None
    plain4, _, pinfo = _run(c, levels, devices=(0,), geo_prior=geo)
    assert bits_equal(plain4, w4) > 0 and pinfo["restored"] is None


@pytest.mark.parametrize("mode", sorted(MODES))
def test_restore_null_equals_gpm_ms_batch_run_prior(mode, monkeypatch):
    from gipuma_b200 import api
    c, photo, geo, (w4, wc, wV, _, _) = _want_prior(mode, "both", 2)
    a4, ac, ainfo = _run(c, 2, devices=(0, 0), planar_prior=photo, geo_prior=geo)
    lib = api.load_library()
    prior = lib.gpm_ms_batch_run_prior
    calls = []

    def via_prior(m, o, v, po, ro, st):
        calls.append(ro)
        return prior(m, o, v, po, st)
    monkeypatch.setattr(lib, "gpm_ms_batch_run_restore", via_prior)
    b4, bc, binfo = _run(c, 2, devices=(0, 0), planar_prior=photo, geo_prior=geo)
    assert calls == [None]
    assert bits_equal(a4, w4) == 0 and bits_equal(ac, wc) == 0 and bits_equal(b4, w4) == 0 and bits_equal(bc, wc) == 0
    assert ainfo["prior"] == binfo["prior"] and ainfo["restored"] is None


@pytest.mark.parametrize("mode", ["pm_fixed", "ncc_adaptive_jvs"])
def test_degenerate_thresholds(mode):
    """threshold 1e30, no restored sweep: no detail pixel, and the planes are the restorer-free run's.  threshold -1e30: every
    pixel with finite costs is a detail pixel; with no sweep the planes are batch_run's with params.iterations =
    photo_iterations.  Costs are not compared: the restorer's are gpm_cost_eval's (the propagation rounding variant) of the
    final planes, while the sweeps store, at pixels whose last accept was a refinement, the refinement variant's."""
    from gipuma_b200 import api
    c = _driver_case(mode)
    H, W = c["images"].shape[1:3]
    plain4, _, _ = _run(c, 2, devices=(0, 0))
    n4, _, info = _run(c, 2, devices=(0, 0), detail_restorer={"threshold": 1e30, "iterations": 0, "photo_iterations": 2})
    assert bits_equal(n4, plain4) == 0 and info["restored"] == [0] * len(c["refs"])
    n4, _, info = _run(c, 2, devices=(0, 0), detail_restorer={"threshold": -1e30, "iterations": 0, "photo_iterations": 3})
    assert info["restored"] == [H * W] * len(c["refs"])
    p = api.GpmParams.from_buffer_copy(api.pack_params(c["params"]))
    p.iterations = 3
    kw = {k: v for k, v in c["modes"].items()}
    b4, _, _ = api.batch_run(c["images"], c["Ps"], p, c["refs"], cam_scale=c["scale"], devices=(0, 0), **KW, **kw)
    assert bits_equal(n4, b4) == 0


def test_dmb_files_equal_the_outputs_and_fuse_and_score(tmp_path):
    from gipuma_b200 import api
    from test_gpu_fusion import FUSE
    c, geo, (w4, _, _, _) = _want_restore("pm_fixed", 3, True)
    refs, Ps = c["refs"], c["Ps"]
    n4, _, _ = _run(c, 3, devices=(0, 0), out_dir=str(tmp_path), geo_prior=geo, detail_restorer=RESTORE)
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


@pytest.mark.parametrize("mode", ["pm_fixed", "ncc_fixed"])
def test_equal_costs_are_not_detail_pixels(mode):
    """One level and no geometric sweep: the geometric stage keeps the coarsest photometric stage's planes, and the
    photometric-only estimate with photo_iterations = params.iterations and the same seed reproduces them, so c_ms == c_ph
    at every pixel.  The comparison is strict: threshold 0 restores nothing, the next float32 below 0 every pixel."""
    from gipuma_b200 import api
    c = _driver_case(mode)
    H, W = c["images"].shape[1:3]
    args = dict(levels=1, geo_iterations=0, cam_scale=c["scale"], jbu=JBU, devices=(0, 0), **KW, **c["modes"])
    plain4, _, _ = api.multiscale_pass(c["images"], c["Ps"], c["params"], c["refs"], **args)
    r = {"photo_iterations": int(c["params"].iterations), "iterations": 0}
    n4, _, info = api.multiscale_pass(c["images"], c["Ps"], c["params"], c["refs"], detail_restorer=dict(r, threshold=0.0), **args)
    assert info["restored"] == [0] * len(c["refs"])
    assert bits_equal(n4, plain4) == 0
    below = float(np.nextafter(f32(0), f32(-1)))
    n4, _, info = api.multiscale_pass(c["images"], c["Ps"], c["params"], c["refs"], detail_restorer=dict(r, threshold=below), **args)
    assert info["restored"] == [H * W] * len(c["refs"])
    assert bits_equal(n4, plain4) == 0                      # every pixel took the estimate's plane, which is the same plane

"""The coarse-to-fine scheme (DESIGN.md §19) on the GPU, every check bit for bit.

- gpm_downsample equals oracle/pyscale.downsample, grey and RGBA, at odd, even and ragged sizes, from host and device memory;
- gpm_upsample_planes equals pyscale.jbu at ragged sizes, radius 0, 2 and 4, grey and colour guides, on adversarial coarse
  states (NaN, out-of-range, behind-camera and all-zero planes); it ignores the context's modes and leaves its state, costs
  and counters as they were;
- gpm_ms_batch_run with one level equals geometric_pass over V; with two and three levels it equals the flow restated here
  through Context calls, api.downsample and Context.upsample_planes, with 1, 2 and 3 workers on one GPU and over every GPU,
  and reports V, the transitive closure of the selections;
- its .dmb files equal its outputs, which fuse and score; a job failing during the run is reported by view, every image
  registration is released, and the next call succeeds."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import bits_equal
from oracle import pyscale

pytestmark = pytest.mark.gpu

KW = dict(min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
GEO_ITERATIONS = 1
JBU = dict(radius=2, sigma_space=2.0, sigma_range=10.0)


# ---- gpm_downsample --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("channels", [1, 4])
@pytest.mark.parametrize("W,H", [(150, 101), (9, 8), (1601, 1201)])
def test_downsample_equals_the_restatement(W, H, channels):
    import torch
    from gipuma_b200 import api
    rng = np.random.default_rng(W * H + channels)
    shape = (H, W) if channels == 1 else (H, W, 4)
    img = rng.uniform(0, 255, shape).astype(np.float32)
    img.flat[::97] = rng.uniform(-1e-39, 1e-39, img.flat[::97].shape).astype(np.float32)        # denormals are kept
    want = pyscale.downsample(img)
    got = api.downsample(img)
    assert got.shape == want.shape and bits_equal(got, want) == 0
    got_dev = api.downsample(torch.from_numpy(img).cuda()).cpu().numpy()
    assert bits_equal(got_dev, want) == 0
    levels = api.pyramid(img, 3)
    assert [a.shape[:2] for a in levels] == [(H, W), ((H + 1) // 2, (W + 1) // 2), ((H + 3) // 4, (W + 3) // 4)]
    assert bits_equal(levels[2], pyscale.downsample(want)) == 0


def test_downsample_reads_a_pitched_image():
    from gipuma_b200 import api
    lib = api.load_library()
    img = np.random.default_rng(5).uniform(0, 255, (21, 40)).astype(np.float32)
    out = np.empty((11, 17), np.float32)
    assert lib.gpm_downsample(0, img.ctypes.data, 40 * 4, 33, 21, 1, out.ctypes.data, 0) == 0
    assert bits_equal(out, pyscale.downsample(img[:, :33])) == 0


# ---- gpm_upsample_planes ---------------------------------------------------------------------------------------------------

def _fine_context(W, H, colour, seed=7):
    """A context at W x H with parameters and a reference (a DTU camera), plus what the restatement needs."""
    from gipuma_b200 import api, scene as S
    p = S.AlgorithmParameters(box_hsize=9, box_vsize=9, iterations=1, n_best=2, cost_comb=S.COMB_BEST_N)
    p.depthMin, p.depthMax = 400.0, 900.0
    Ps = S.load_dtu_projections()[:3]
    cams = api.prepare_cameras(Ps, 1600.0 / W)
    rng = np.random.default_rng(seed)
    img = rng.uniform(0, 255, (H, W, 4) if colour else (H, W)).astype(np.float32)
    img = np.where(rng.random(img.shape) < 0.3, np.float32(128), img).astype(np.float32)    # ties in the guide
    ctx = api.Context(W, H, 2)
    ctx.set_params(p)
    ctx.set_reference(img, cams[0])
    return ctx, img, cams, p


def _coarse_state(W, H, cams, p, seed):
    """Random in-range planes with adversarial entries: NaN, out of range, behind the camera, all zero."""
    Wc, Hc = (W + 1) // 2, (H + 1) // 2
    rng = np.random.default_rng(seed)
    n = rng.normal(size=(Hc, Wc, 3))
    n[..., 2] = -np.abs(n[..., 2]) - 1.0
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    Kinv = np.asarray(cams[0].K_inv[:], np.float64).reshape(3, 3)
    ys, xs = np.mgrid[0:Hc, 0:Wc]
    r = np.stack([2 * xs, 2 * ys, np.ones_like(xs)], -1) @ Kinv.T
    depth = rng.uniform(p.depthMin, p.depthMax, (Hc, Wc))
    d = -(n * r * depth[..., None]).sum(-1)
    planes = np.concatenate([n, d[..., None]], -1).astype(np.float32)
    kind = rng.integers(0, 10, (Hc, Wc))
    planes[kind == 0] = np.nan
    planes[kind == 1, 3] *= 5                                   # out of range
    planes[kind == 2, 3] *= -1                                  # behind the camera
    planes[kind == 3] = 0.0
    planes[:2, :3] = 0.0                                        # a block with no usable candidate at radius 0 .. 1
    return planes


def _restated_jbu(ctx, img, cams, p, coarse, radius):
    return pyscale.jbu(coarse, img, np.asarray(cams[0].K_inv[:], np.float32), p.depthMin, p.depthMax, radius,
                       JBU["sigma_space"], JBU["sigma_range"])


@pytest.mark.parametrize("colour", [False, True], ids=["grey", "colour"])
@pytest.mark.parametrize("W,H", [(150, 101), (64, 48), (33, 17)])
@pytest.mark.parametrize("radius", [0, 2, 4])
def test_upsample_planes_equals_the_restatement(W, H, colour, radius):
    ctx, img, cams, p = _fine_context(W, H, colour)
    with ctx:
        coarse = _coarse_state(W, H, cams, p, seed=W + radius)
        want_p, want_d = _restated_jbu(ctx, img, cams, p, coarse, radius)
        got_p, got_d = ctx.upsample_planes(coarse, radius=radius, sigma_space=JBU["sigma_space"], sigma_range=JBU["sigma_range"])
        assert bits_equal(got_p, want_p) == 0 and bits_equal(got_d, want_d) == 0
        assert (want_d > 0).any() and (radius > 0 or (want_d == 0).any())
    import torch
    ctx, img, cams, p = _fine_context(W, H, colour)
    with ctx:
        dp, dd = ctx.upsample_planes(torch.from_numpy(coarse).cuda(), radius=radius, **{k: JBU[k] for k in ("sigma_space", "sigma_range")})
        assert bits_equal(dp.cpu().numpy(), want_p) == 0 and bits_equal(dd.cpu().numpy(), want_d) == 0


def test_upsample_planes_ignores_modes_and_leaves_the_state_alone():
    from gipuma_b200 import api
    W, H = 96, 64
    ctx, img, cams, p = _fine_context(W, H, False)
    coarse = _coarse_state(W, H, cams, p, seed=3)
    want_p, want_d = _restated_jbu(ctx, img, cams, p, coarse, 2)
    with ctx:
        ctx.set_view(0, img, cams[1])
        ctx.set_num_views(1)
        ctx.set_view_depth(0, np.full((H, W), 600.0, np.float32))
        ctx.set_rng(11)
        ctx.init()
        s4, sc = ctx.get_state()
        ctx.reset_stats()
        st = ctx.stats()
        for mode in ("plain", "geometric", "jvs"):
            if mode == "geometric":
                ctx.set_geometric(0.5, 3.0)
            if mode == "jvs":
                ctx.set_geometric(0.0, 3.0)
                ctx.set_photometric("ncc")
                ctx.set_view_selection("joint")
            got_p, got_d = ctx.upsample_planes(coarse, **JBU)
            assert bits_equal(got_p, want_p) == 0 and bits_equal(got_d, want_d) == 0, mode
            a4, ac = ctx.get_state()
            assert bits_equal(a4, s4) == 0 and bits_equal(ac, sc) == 0 and ctx.stats() == st, mode


def test_upsample_planes_refuses_without_parameters_or_reference():
    from gipuma_b200 import api
    with api.Context(32, 16, 1) as ctx:
        with pytest.raises(api.GipumaError, match="-3"):
            ctx.upsample_planes(np.zeros((8, 16, 4), np.float32))
        lib, jbu = ctx.lib, api.jbu_params()
        c = np.zeros((8, 16, 4), np.float32)
        assert lib.gpm_upsample_planes(ctx.h, c.ctypes.data, 15, 8, 0, C.byref(jbu), None, None) == -1


# ---- gpm_ms_batch_run ------------------------------------------------------------------------------------------------------

def _closure(Ps, refs, W, H, cam_scale, min_angle, max_angle, max_views):
    from gipuma_b200 import api
    n = len(Ps)
    plan, todo = {}, list(dict.fromkeys(refs))
    while todo:
        r = todo.pop(0)
        if r in plan:
            continue
        order = [r] + [i for i in range(n) if i != r]
        cams = api.prepare_cameras([Ps[i] for i in order], cam_scale)
        subset, rng = api.select_views(cams, W, H, min_angle, max_angle, max_views)
        assert subset
        plan[r] = (order, subset, rng)
        todo += [order[k] for k in subset if order[k] not in plan]
    return plan


def _restated(images, Ps, params, refs, levels, cam_scale, min_angle, max_angle, max_views, seed, weight, max_err, jbu,
              photometric="pm", propagation="fixed", view_selection="off"):
    """The multi-level flow through one Context per level, view by view in ascending order."""
    from gipuma_b200 import api
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

    ctxs = [api.Context(w, h, max_views) for w, h in size]
    out = {}
    try:
        top = levels - 1
        raw, depth = {}, {}
        for i in V:
            load(ctxs[top], top, i)
            ctxs[top].init()
            ctxs[top].sweep(params.iterations)
            raw[i] = ctxs[top].get_state()[0]
            ctxs[top].finalize()
            depth[i] = np.ascontiguousarray(ctxs[top].get_state()[0][..., 3])
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
                if l > 0:
                    new_raw[i] = ctx.get_state()[0]
                else:
                    ctx.finalize()
                    out[i] = ctx.get_state()
                ctx.set_geometric(0.0, max_err)
            raw = new_raw
    finally:
        for c in ctxs:
            c.close()
    n4 = np.stack([out[r][0] for r in refs])
    cc = np.stack([out[r][1] for r in refs])
    return n4, cc, V


CASES = {
    "fusion_pm_grey": dict(name="fusion", colour=False),
    "ragged_pm_colour": dict(name="ragged", colour=True),
    "ragged_ncc_grey": dict(name="ragged", colour=False, photometric="ncc"),
    "fusion_ncc_adaptive_jvs": dict(name="fusion", colour=False, photometric="ncc", propagation="adaptive", view_selection="joint"),
}
_CACHE = {}


def _want(case, levels):
    from gipuma_b200 import api
    from test_gpu_geometric_batch import _case
    key = (case, levels)
    if key not in _CACHE:
        spec = dict(CASES[case])
        c = _case(spec.pop("name"), spec.pop("colour"))
        c["modes"] = spec
        _CACHE[key] = (c, _restated(c["images"], c["Ps"], c["params"], c["refs"], levels, c["scale"], weight=api.GEO_WEIGHT,
                                    max_err=api.GEO_MAX_ERR, jbu=JBU, **KW, **spec))
    return _CACHE[key]


def _run(c, levels, **kw):
    from gipuma_b200 import api
    return api.multiscale_pass(c["images"], c["Ps"], c["params"], c["refs"], levels=levels, geo_iterations=GEO_ITERATIONS,
                               cam_scale=c["scale"], jbu=JBU, **KW, **c["modes"], **kw)


def _device_lists():
    import torch
    lists = [(0,), (0, 0), (0, 0, 0)]
    if torch.cuda.device_count() > 1:
        lists.append(tuple(range(torch.cuda.device_count())))
    return lists


@pytest.mark.parametrize("levels", [2, 3])
@pytest.mark.parametrize("case", sorted(CASES))
def test_driver_equals_the_restated_multilevel_flow(case, levels):
    c, (w4, wc, wV) = _want(case, levels)
    for devices in _device_lists():
        n4, cost, info = _run(c, levels, devices=devices)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (case, levels, devices)
        assert info["views"] == wV, devices
        assert len(info["level_sweep_s"]) == levels and all(t > 0 for t in info["level_sweep_s"])
        assert all(t > 0 for t in info["level_upsample_s"][:levels - 1]) and info["level_upsample_s"][levels - 1] == 0
        assert all(d in devices for d in info["device"])


def test_views_are_the_transitive_closure():
    from gipuma_b200 import api
    from test_gpu_geometric_batch import _case
    c = _case("ragged", False)
    refs = [7]
    _, _, info = api.multiscale_pass(c["images"], c["Ps"], c["params"], refs, levels=2, geo_iterations=GEO_ITERATIONS,
                                     cam_scale=c["scale"], jbu=JBU, **KW)
    H, W = c["images"].shape[1:3]
    plan = _closure(c["Ps"], refs, W, H, c["scale"], KW["min_angle"], KW["max_angle"], KW["max_views"])
    one_step = set(refs) | {plan[7][0][k] for k in plan[7][1]}
    assert info["views"] == sorted(plan)
    assert set(info["views"]) >= one_step


@pytest.mark.parametrize("colour", [False, True], ids=["grey", "colour"])
def test_one_level_is_the_geometric_pass_over_the_view_set(colour):
    from gipuma_b200 import api
    from test_gpu_geometric_batch import _case
    c = _case("ragged", colour)
    n4, cost, info = api.multiscale_pass(c["images"], c["Ps"], c["params"], c["refs"], levels=1, geo_iterations=GEO_ITERATIONS,
                                         cam_scale=c["scale"], devices=(0, 0), **KW)
    V = info["views"]
    g4, gc, ginfo = api.geometric_pass(c["images"], c["Ps"], c["params"], V, geo_iterations=GEO_ITERATIONS, cam_scale=c["scale"],
                                       devices=(0, 0), **KW)
    assert ginfo["pass1_views"] == V
    rows = [V.index(r) for r in c["refs"]]
    assert bits_equal(n4, g4[rows]) == 0 and bits_equal(cost, gc[rows]) == 0


def test_dmb_files_equal_the_outputs_and_fuse_and_score(tmp_path):
    from gipuma_b200 import api
    from test_gpu_fusion import FUSE
    c, (w4, _, _) = _want("fusion_pm_grey", 3)
    refs, Ps = c["refs"], c["Ps"]
    n4, _, _ = _run(c, 3, devices=(0, 0), out_dir=str(tmp_path))
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


def test_failure_during_the_run_is_named_and_releases_the_image_registrations():
    import torch
    from gipuma_b200 import api
    from test_gpu_geometric_batch import _case
    c = _case("ragged", False)
    images = c["images"]
    assert images.dtype == np.float32 and images.flags["C_CONTIGUOUS"]          # the driver registers these very buffers
    bad = c["params"]
    bad_iterations, bad.iterations = bad.iterations, -1
    try:
        with pytest.raises(api.GipumaError, match=r"level 1 photometric stage of view \d+"):
            api.multiscale_pass(images, c["Ps"], bad, c["refs"], levels=2, geo_iterations=GEO_ITERATIONS, cam_scale=c["scale"],
                                devices=(0, 0), jbu=JBU, **KW)
    finally:
        bad.iterations = bad_iterations
    cudart = torch.cuda.cudart()
    for i in range(len(images)):
        ptr = images[i].ctypes.data
        assert int(cudart.cudaHostRegister(ptr, images[i].nbytes, 1)) == 0, i
        assert int(cudart.cudaHostUnregister(ptr)) == 0, i
    c2 = dict(c, modes={})
    n4, _, _ = _run(c2, 2, devices=(0, 0))
    assert np.all(np.isfinite(n4))

"""The two-pass geometric-consistency batch driver (gpm_geo_batch_run, DESIGN.md §14) on the GPU.

- Its norm4 and cost equal, bit for bit, the two-pass flow restated here through Context calls (the single-context Python
  loop the driver replaced), grey and colour, on the fusion test's dataset and at a ragged size, with one, two and three
  workers on one GPU and with every visible GPU;
- it reports the pass-1 views (the closure of the references' selections, ascending) and each reference's selected views;
- its .dmb files equal its in-memory outputs and fuse to the same vertices;
- a reference view without source views is refused by name while the driver plans, before it registers an image, allocates
  its host store or creates a context; the next call on the same images succeeds;
- a job that fails during the run (gpm_set_params refuses a negative iteration count in pass 1) stops the call with the view
  named, and every image is unregistered again: the test can page-lock it itself afterwards."""
import os

import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu

KW = dict(min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
GEO_ITERATIONS = 1


def _colour(grey):
    """RGBA images whose channels are fixed functions of the grey value (as scene.colorize makes them)."""
    g = grey.astype(np.float64)
    gr = np.clip(np.rint(245.0 - 0.85 * g), 0, 255)
    r = np.clip(np.rint(127.5 + 110.0 * np.sin(g / 23.0)), 0, 255)
    return np.ascontiguousarray(np.stack([g, gr, r, np.zeros_like(g)], axis=-1), dtype=np.float32)


def _case(name, colour):
    from gipuma_b200 import scene as S
    from test_gpu_fusion import REFS, _dataset, _params
    if name == "fusion":                                   # 24 DTU cameras at 128x96, 8 reference views
        Ps, scale, images, hf = _dataset()
        refs = REFS
    else:                                                  # ragged: 10 cameras at 150x101, 3 reference views
        Ps, scale, images, hf = _dataset(rows=101, cols=150, n_cams=10)
        refs = [7, 0, 4]
    p = _params()
    p.iterations = 2
    return dict(Ps=Ps, scale=scale, images=_colour(images) if colour else images, refs=refs, params=p, hf=hf)


def _restated(images, Ps, params, refs, cam_scale, min_angle, max_angle, max_views, seed, weight, max_err):
    """The two-pass flow through one Context: pass 1 over the references and the views they select, in that order, then
    pass 2 per reference view."""
    from gipuma_b200 import api
    import ctypes as C
    n, H, W = images.shape[:3]

    def load_job(ctx, ref):
        order = [ref] + [i for i in range(n) if i != ref]
        cams = api.prepare_cameras([Ps[i] for i in order], cam_scale)
        subset, (lo, hi) = api.select_views(cams, W, H, min_angle, max_angle, max_views)
        assert subset
        p = api.GpmParams.from_buffer_copy(api.pack_params(params))
        p.depthMin = p.depthMin if p.depthMin > 0 else lo
        p.depthMax = p.depthMax if p.depthMax > 0 else hi
        fb = np.float32(cams[0].f) * np.float32(cams[0].baseline)
        p.min_disparity, p.max_disparity = float(fb / np.float32(p.depthMax)), float(fb / np.float32(p.depthMin))
        ctx._check(ctx.lib.gpm_set_params(ctx.h, C.byref(p)))
        ctx.set_reference(images[ref], cams[0])
        for v, k in enumerate(subset):
            ctx.set_view(v, images[order[k]], cams[k])
        ctx.set_num_views(len(subset))
        ctx.set_rng(seed, api.GPM_RNG_REFERENCE)
        return [order[k] for k in subset]

    n4 = np.empty((len(refs), H, W, 4), np.float32)
    cc = np.empty((len(refs), H, W), np.float32)
    views = []
    with api.Context(W, H, max_views) as ctx:
        sources, raw, depth = {}, {}, {}
        todo = list(dict.fromkeys(refs))
        while todo:
            r = todo.pop(0)
            if r in depth:
                continue
            sources[r] = load_job(ctx, r)
            ctx.init()
            ctx.sweep(params.iterations)
            if r in refs:
                raw[r] = ctx.get_state()[0]
            ctx.finalize()
            depth[r] = np.ascontiguousarray(ctx.get_state()[0][..., 3])
            if r in refs:
                todo += [i for i in sources[r] if i not in depth]
        for j, r in enumerate(refs):
            src = load_job(ctx, r)
            for v, i in enumerate(src):
                ctx.set_view_depth(v, depth[i])
            ctx.set_geometric(weight, max_err)
            ctx.set_state(raw[r], ctx.cost_eval(raw[r]))
            ctx.sweep(GEO_ITERATIONS)
            ctx.finalize()
            n4[j], cc[j] = ctx.get_state()
            ctx.set_geometric(0.0, max_err)
            views.append(src)
    return n4, cc, sorted(depth), views


_CACHE = {}


def _want(name, colour):
    from gipuma_b200 import api
    if (name, colour) not in _CACHE:
        c = _case(name, colour)
        _CACHE[(name, colour)] = (c, _restated(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], weight=api.GEO_WEIGHT,
                                               max_err=api.GEO_MAX_ERR, **KW))
    return _CACHE[(name, colour)]


def _device_lists():
    import torch
    lists = [(0,), (0, 0), (0, 0, 0)]
    if torch.cuda.device_count() > 1:
        lists.append(tuple(range(torch.cuda.device_count())))
    return lists


@pytest.mark.parametrize("colour", [False, True], ids=["grey", "colour"])
@pytest.mark.parametrize("name", ["fusion", "ragged"])
def test_driver_equals_the_restated_two_pass_flow(name, colour):
    from gipuma_b200 import api
    c, (w4, wc, w_pass1, w_views) = _want(name, colour)
    for devices in _device_lists():
        n4, cost, info = api.geometric_pass(c["images"], c["Ps"], c["params"], c["refs"], geo_iterations=GEO_ITERATIONS,
                                            cam_scale=c["scale"], devices=devices, **KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (name, colour, devices)
        assert info["pass1_views"] == w_pass1 and info["views"] == w_views, devices
        assert len(info["pass1_sweep_s"]) == len(w_pass1) and len(info["pass2_sweep_s"]) == len(c["refs"])
        assert all(t > 0 for t in info["pass1_sweep_s"] + info["pass2_sweep_s"])
        assert all(d in devices for d in info["device"])


def test_selected_views_are_the_view_selection_subsets():
    from gipuma_b200 import api
    c, (_, _, w_pass1, _) = _want("ragged", False)
    _, _, info = api.geometric_pass(c["images"], c["Ps"], c["params"], c["refs"], geo_iterations=GEO_ITERATIONS,
                                    cam_scale=c["scale"], **KW)
    n, H, W = c["images"].shape
    closure = set(c["refs"])
    for j, ref in enumerate(c["refs"]):
        order = [ref] + [i for i in range(n) if i != ref]
        cams = api.prepare_cameras([c["Ps"][i] for i in order], c["scale"])
        subset, _ = api.select_views(cams, W, H, KW["min_angle"], KW["max_angle"], KW["max_views"])
        assert info["views"][j] == [order[k] for k in subset]
        closure |= set(info["views"][j])
    assert info["pass1_views"] == sorted(closure) == w_pass1


def test_dmb_files_equal_the_outputs_and_fuse_alike(tmp_path):
    from gipuma_b200 import api
    from test_gpu_fusion import FUSE
    c, _ = _want("fusion", False)
    refs, Ps = c["refs"], c["Ps"]
    n4, _, _ = api.geometric_pass(c["images"], Ps, c["params"], refs, geo_iterations=GEO_ITERATIONS, cam_scale=c["scale"],
                                  devices=(0, 0), out_dir=str(tmp_path), **KW)
    for j, ref in enumerate(refs):
        d = api.read_dmb(os.path.join(str(tmp_path), "%08d" % ref, "disp.dmb"))
        nm = api.read_dmb(os.path.join(str(tmp_path), "%08d" % ref, "normals.dmb"))
        assert bits_equal(d, n4[j][..., 3]) == 0 and bits_equal(nm, n4[j][..., :3]) == 0
    v_mem, _ = api.fuse(n4, [Ps[r] for r in refs], cam_scale=c["scale"], **FUSE)
    v_dir, _ = api.fuse_batch_dir(str(tmp_path), refs, Ps, cam_scale=c["scale"], **FUSE)
    assert len(v_mem) > 1000 and v_mem.tobytes() == v_dir.tobytes()


def test_reference_without_source_views_is_refused_by_name_while_planning():
    from gipuma_b200 import api
    c, _ = _want("ragged", False)
    flipped = c["Ps"][0] @ np.diag([-1.0, 1.0, -1.0, 1.0])      # looks away from the scene: no camera within 5 .. 45 degrees
    Ps = list(c["Ps"]) + [flipped]
    images = np.concatenate([c["images"], c["images"][:1]])
    bad = len(Ps) - 1
    with pytest.raises(api.GipumaError, match="reference view %d$" % bad):
        api.geometric_pass(images, Ps, c["params"], [0, bad, 4], geo_iterations=GEO_ITERATIONS, cam_scale=c["scale"],
                           devices=(0, 0), **KW)
    n4, _, info = api.geometric_pass(images, Ps, c["params"], [0, 4], geo_iterations=GEO_ITERATIONS, cam_scale=c["scale"],
                                     devices=(0, 0), **KW)
    assert bad not in info["pass1_views"] and np.all(np.isfinite(n4))


def test_failure_during_the_run_releases_the_image_registrations():
    import torch
    from gipuma_b200 import api
    c, _ = _want("ragged", False)
    images = c["images"]
    assert images.dtype == np.float32 and images.flags["C_CONTIGUOUS"]          # the driver registers these very buffers
    bad = c["params"]
    bad_iterations, bad.iterations = bad.iterations, -1
    try:
        with pytest.raises(api.GipumaError, match="pass 1 of view"):
            api.geometric_pass(images, c["Ps"], bad, c["refs"], geo_iterations=GEO_ITERATIONS, cam_scale=c["scale"],
                               devices=(0, 0), **KW)
    finally:
        bad.iterations = bad_iterations
    cudart = torch.cuda.cudart()
    for i in range(len(images)):                 # still registered by the driver: cudaErrorHostMemoryAlreadyRegistered
        ptr = images[i].ctypes.data
        assert int(cudart.cudaHostRegister(ptr, images[i].nbytes, 1)) == 0, i
        assert int(cudart.cudaHostUnregister(ptr)) == 0, i
    n4, _, _ = api.geometric_pass(images, c["Ps"], c["params"], c["refs"], geo_iterations=GEO_ITERATIONS, cam_scale=c["scale"],
                                  devices=(0, 0), **KW)
    assert bits_equal(n4, _want("ragged", False)[1][0]) == 0

"""The NCC photometric cost (DESIGN.md §15) without a GPU: the numpy restatement's known answers, the summation order it
pins, and the argument refusals of the Python API and of the C-ABI's batch drivers, all before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

from test_geo_batch_args import _desc

f32 = np.float32
E_ARG, E_STATE = -1, -3


def ncc(w, r, t, min_std=1.0):
    from oracle import pyncc
    return pyncc.ncc_cost(np.asarray(w, f32), np.asarray(r, f32), np.asarray(t, f32), min_std)


def test_identical_patches_cost_zero():
    rng = np.random.default_rng(1)
    w = rng.uniform(0.05, 1.0, (500, 64)).astype(f32)
    r = rng.uniform(0, 255, (500, 64)).astype(f32)
    assert np.all(ncc(w, r, r) == 0)


def test_gain_and_offset_cost_zero():
    rng = np.random.default_rng(2)
    w = rng.uniform(0.05, 1.0, (1000, 64)).astype(f32)
    r = rng.integers(0, 256, (1000, 64)).astype(f32)
    for a, b in ((1.25, -17.0), (0.75, 40.0), (1.5, 3.0)):       # t = a r + b exactly
        c = ncc(w, r, (f32(a) * r + f32(b)).astype(f32))
        # the one-pass variances lose a few bits to cancellation (mean^2 / variance ~ 4 here): 31 ulp of 1 measured
        assert np.all(c <= 64 * np.finfo(f32).eps) and (c == 0).mean() > 0.3, (a, b, c.max())
    # every step exact: W = 4, r = 1, 3, 5, 7 (mean 4, variance 5), t = 2 r + 3 (mean 11, variance 20, covariance 10)
    assert ncc([1, 1, 1, 1], [1, 3, 5, 7], [5, 9, 13, 17]) == 0


def test_negative_gain_costs_two():
    r = np.array([1, 3, 5, 7], f32)
    assert ncc([1, 1, 1, 1], r, -2 * r + 40) == 2
    rng = np.random.default_rng(3)
    w = rng.uniform(0.05, 1.0, (200, 64)).astype(f32)
    r = rng.uniform(0, 255, (200, 64)).astype(f32)
    assert np.all(np.abs(ncc(w, r, (f32(-0.7) * r + f32(200)).astype(f32)) - 2) <= 64 * np.finfo(f32).eps)


def test_flat_windows_and_the_variance_floor():
    w = [1, 1]
    assert ncc(w, [5, 5], [1, 9]) == 2                           # flat reference window
    assert ncc(w, [1, 9], [7, 7]) == 2                           # flat source window
    # r = 0, 2: mean 1, variance exactly 1 = min_std^2: the window counts
    assert ncc(w, [0, 2], [0, 2], min_std=1.0) == 0
    assert ncc(w, [0, 2], [2, 0], min_std=1.0) == 2              # anti-correlated
    # the same variance just below the floor
    assert ncc(w, [0, 2], [0, 2], min_std=np.nextafter(f32(1), f32(2))) == 2
    assert ncc(w, [0, 2], [0, 4], min_std=np.nextafter(f32(1), f32(2))) == 2
    assert ncc([0, 0], [1, 9], [1, 9]) == 2                      # no weight at all


def _scalar_cost(w, r, t, min_std):
    """§15 with float32 scalars, sample after sample (an independent restatement of the specified order)."""
    W = Sr = Srr = St = Stt = Srt = f32(0)
    for ws, rs, ts in zip(w, r, t):
        a = f32(ws * rs)
        W, Sr, Srr = f32(W + ws), f32(Sr + a), f32(Srr + f32(a * rs))
        wt = f32(ws * ts)
        St, Stt, Srt = f32(St + wt), f32(Stt + f32(wt * ts)), f32(Srt + f32(a * ts))
    mr, mt = f32(Sr / W), f32(St / W)
    vr, vt = f32(f32(Srr / W) - f32(mr * mr)), f32(f32(Stt / W) - f32(mt * mt))
    c = f32(f32(Srt / W) - f32(mr * mt))
    s2 = f32(f32(min_std) * f32(min_std))
    if not (W > 0 and vr >= s2 and vt >= s2):
        return f32(2)
    x = f32(f32(1) - f32(c / np.sqrt(f32(vr * vt))))
    return f32(2) if np.isnan(x) else min(f32(2), max(f32(0), x))


def test_summation_order_is_pinned():
    """On windows where the reversed sample order gives other bits, the restatement gives the sequential order's."""
    rng = np.random.default_rng(4)
    found = 0
    for _ in range(400):
        w = rng.uniform(0.01, 1.0, 64).astype(f32)
        r = rng.uniform(0, 255, 64).astype(f32)
        t = (r * f32(0.8) + rng.normal(0, 20, 64)).astype(f32)
        want = _scalar_cost(w, r, t, 2.0)
        if want == _scalar_cost(w[::-1], r[::-1], t[::-1], 2.0):
            continue
        found += 1
        assert ncc(w, r, t, 2.0).view(np.uint32) == want.view(np.uint32)
    assert found >= 20, found


def test_sums_flush_denormals_like_the_device():
    from oracle import pyncc
    tiny = np.finfo(f32).tiny
    Ws, Sr, Srr = pyncc.window_sums(np.array([[tiny]], f32), np.array([[f32(0.25)]], f32))
    assert Ws[0] == tiny and Sr[0] == 0 and Srr[0] == 0             # tiny * 0.25 is a denormal: flushed


@pytest.mark.parametrize("kw", [dict(photometric="census"), dict(photometric="ncc", ncc_min_std=0.0),
                                dict(photometric="ncc", ncc_min_std=float("nan")), dict(photometric="ncc", ncc_min_std=-1.0),
                                dict(photometric="ncc", ncc_min_std=float("inf"))])
@pytest.mark.parametrize("entry", ["batch_run", "geometric_pass"])
def test_api_refuses_bad_arguments_before_loading_the_library(monkeypatch, kw, entry):
    from gipuma_b200 import api, scene as S

    def no_library():
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(api, "load_library", no_library)
    params = S.AlgorithmParameters(box_hsize=9, box_vsize=9, iterations=1)
    imgs = np.zeros((3, 16, 16), np.float32)
    with pytest.raises(ValueError):
        getattr(api, entry)(imgs, [np.eye(3, 4)] * 3, params, [0], **kw)


def test_geometric_pass_refuses_ncc_on_colour_images_before_loading_the_library(monkeypatch):
    from gipuma_b200 import api, scene as S
    monkeypatch.setattr(api, "load_library", lambda: (_ for _ in ()).throw(AssertionError("the library was loaded")))
    params = S.AlgorithmParameters(box_hsize=9, box_vsize=9, iterations=1)
    with pytest.raises(ValueError, match="grey"):
        api.geometric_pass(np.zeros((3, 16, 16, 4), np.float32), [np.eye(3, 4)] * 3, params, [0], photometric="ncc")
    assert api.check_photometric("pm", float("nan")) == 0           # min_std is ignored for the PM cost


@pytest.mark.parametrize("kind,min_std,channels,msg", [(2, 1.0, 1, "kind"), (-1, 1.0, 1, "kind"), (1, 0.0, 1, "min_std"),
                                                       (1, float("nan"), 1, "min_std"), (1, float("inf"), 1, "min_std"),
                                                       (1, -3.0, 1, "min_std"), (1, 2.0, 4, "grey")])
def test_photo_drivers_refuse_bad_arguments_without_a_device(kind, min_std, channels, msg):
    from gipuma_b200 import api
    lib = api.load_library()
    g, _keep = _desc(channels=channels)
    rc = lib.gpm_geo_batch_run_photo(C.byref(g), kind, min_std, None)
    err = lib.gpm_batch_last_error().decode()
    assert rc == E_ARG and err.startswith("gpm_geo_batch_run_photo: bad arguments") and msg in err, (rc, err)
    if channels == 1:
        rc = lib.gpm_batch_run_photo(C.byref(g.batch), kind, min_std, None)
        err = lib.gpm_batch_last_error().decode()
        assert rc == E_ARG and err.startswith("gpm_batch_run_photo: bad arguments") and msg in err, (rc, err)


def test_photo_drivers_refuse_bad_descriptors_without_a_device():
    from gipuma_b200 import api
    lib = api.load_library()
    assert lib.gpm_batch_run_photo(None, 0, 0.0, None) == E_ARG
    assert lib.gpm_geo_batch_run_photo(None, 1, 2.0, None) == E_ARG
    g, _keep = _desc(max_views=0)
    assert lib.gpm_geo_batch_run_photo(C.byref(g), 1, 2.0, None) == E_ARG
    assert lib.gpm_batch_run_photo(C.byref(g.batch), 1, 2.0, None) == E_ARG
    assert lib.gpm_batch_last_error().decode() == "gpm_batch_run_photo: bad arguments"


def test_pm_on_colour_images_passes_the_argument_checks():
    """PM with colour images (min_std ignored) is the geometric driver's ordinary case: its arguments are accepted, and the
    call is refused only later, while planning and still before any CUDA call, for a view without source views."""
    from gipuma_b200 import api, scene as S
    lib = api.load_library()
    params = S.AlgorithmParameters(box_hsize=9, box_vsize=9, iterations=1, n_best=2, cost_comb=S.COMB_BEST_N)
    params.depthMin, params.depthMax = 300.0, 800.0
    Ps = [S.load_dtu_projections()[i] for i in range(3)]
    imgs = np.zeros((3, 64, 96, 4), np.float32)                    # RGBA images: what channels = 4 reads
    d, keep = api._batch_desc(imgs, Ps, params, [0, 2], (0,), 1600.0 / 96, 0.1, 0.2, 2, 7, None, None, None)
    g = api.GpmGeoBatchDesc(d, 4, 1, 0.5, 3.0)                     # no camera within 0.1 .. 0.2 degrees of another
    rc = lib.gpm_geo_batch_run_photo(C.byref(g), 0, float("nan"), None)
    err = lib.gpm_batch_last_error().decode()
    assert rc == E_STATE and err.startswith("gpm_geo_batch_run_photo: no source view") and err.endswith("reference view 0"), (rc, err)
    rc = lib.gpm_geo_batch_run_photo(C.byref(g), 1, 2.0, None)      # the same descriptor with NCC: refused for its arguments
    assert rc == E_ARG and "grey" in lib.gpm_batch_last_error().decode()

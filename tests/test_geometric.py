"""The geometric-consistency term (DESIGN.md §14) without a GPU: the numpy restatement (oracle/pygeo.py) gives the known
answers on hand-made cameras, and the new entry points refuse bad arguments before any CUDA call."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest

f32 = np.float32
H, W = 24, 64
FX, CX, CY = 512.0, 31.0, 11.0         # every camera quantity below is a binary fraction: the restated steps are exact
Z0 = 4.0


def cam(tx=0.0, ty=0.0, tz=0.0):
    K = np.array([[FX, 0, CX], [0, FX, CY], [0, 0, 1]])
    return SimpleNamespace(K=K.astype(f32), K_inv=np.linalg.inv(K).astype(f32), R=np.eye(3, dtype=f32),
                           t=np.array([tx, ty, tz], f32))


def fronto_parallel(depth):
    """Planes n = (0, 0, -1), d = depth: the points at that depth along every ray."""
    pl = np.zeros((H, W, 4), f32)
    pl[..., 2] = -1.0
    pl[..., 3] = depth
    return pl


def g(planes, view, depth, weight=0.5, max_err=100.0, lo=1.0, hi=100.0):
    from oracle import pygeo
    return pygeo.geo_cost(planes, cam(), view, np.broadcast_to(f32(depth), (H, W)), weight, max_err, lo, hi)


def test_identical_views_with_consistent_depths_give_zero_error():
    out = g(fronto_parallel(Z0), cam(), Z0)
    assert out.dtype == np.float32 and np.all(out.view(np.uint32) == 0)


@pytest.mark.parametrize("scale", [2.0, 0.5, 1.25])
def test_scaled_depth_gives_the_analytic_pixel_error(scale):
    # view j sits 0.25 to the right: a point at depth 4 appears 512 * 0.25 / 4 = 32 px further left, so u' = px - 32; read
    # back at depth s * 4 along that ray it reprojects to u' + 32 / s, i.e. 32 (1/s - 1) px from p, on the same row
    shift = FX * 0.25 / Z0
    out = g(fronto_parallel(Z0), cam(tx=-0.25), scale * Z0, weight=0.5)
    err = abs(shift * (1.0 / scale - 1.0))
    inside = out[:, int(shift):]
    np.testing.assert_allclose(inside, 0.5 * err, rtol=1e-6, atol=0)
    assert np.all(out[:, :int(shift)] == f32(0.5) * f32(100.0))          # u' < 0: off-image
    capped = g(fronto_parallel(Z0), cam(tx=-0.25), scale * Z0, weight=0.5, max_err=err / 2)
    assert np.all(capped[:, int(shift):] == f32(0.5) * f32(err / 2))


@pytest.mark.parametrize("depth", [0.0, 0.5, 250.0, np.nan])
def test_invalid_depth_gives_weight_times_max_err(depth):
    out = g(fronto_parallel(Z0), cam(), depth, weight=0.25, max_err=3.0)
    assert np.all(out == f32(0.25) * f32(3.0))


def test_points_off_image_or_behind_a_camera_give_weight_times_max_err():
    far = f32(0.25) * f32(3.0)
    # off-image: view j shifted by a whole image width
    assert np.all(g(fronto_parallel(Z0), cam(tx=-1.0), Z0, weight=0.25, max_err=3.0) == far)
    # behind the reference: the plane's point on the ray has negative depth
    assert np.all(g(fronto_parallel(-Z0), cam(), Z0, weight=0.25, max_err=3.0) == far)
    # behind view j: its centre lies 10 in front of the reference, past the points at depth 4
    assert np.all(g(fronto_parallel(Z0), cam(tz=-10.0), Z0, weight=0.25, max_err=3.0) == far)


def test_weight_zero_adds_nothing():
    out = g(fronto_parallel(Z0), cam(tx=-0.25), 2 * Z0, weight=0.0)
    assert np.all(out.view(np.uint32) == 0)


def test_combination_restatement_known_answers():
    from oracle import pygeo
    c = np.array([[[3.0]], [[1.0]], [[2000.0]], [[2.0]]], f32)          # one pixel, four views, one invalid
    assert pygeo.combine(c, 1, 2, 1.5, {2: 0.5})[0, 0] == f32(1.5)      # best_n = 2: (1 + 2) / 2
    assert pygeo.combine(c, 0, 2, 1.5, {3: f32(1) / f32(3)})[0, 0] == (f32(1) + f32(2) + f32(3)) * (f32(1) / f32(3))
    # good: all four, each capped at 1.5 x the smallest, MAXCOST included
    assert pygeo.combine(c, 3, 2, 1.5, {4: 0.25})[0, 0] == (f32(1) + f32(1.5) + f32(1.5) + f32(1.5)) * f32(0.25)
    assert pygeo.combine(np.full((2, 1, 1), 1e4, f32), 1, 2, 1.5, {})[0, 0] == f32(1000.0)   # no valid view


@pytest.mark.parametrize("weight,max_err", [(-0.1, 1.0), (float("nan"), 1.0), (float("inf"), 1.0),
                                            (1.0, 0.0), (1.0, -1.0), (1.0, float("nan")), (1.0, float("inf"))])
def test_bad_geometric_arguments_are_refused_before_any_cuda_call(monkeypatch, weight, max_err):
    from gipuma_b200 import api

    def no_context(*a, **k):
        raise AssertionError("a context was created for arguments that must be refused")
    monkeypatch.setattr(api, "Context", no_context)
    with pytest.raises(ValueError):
        api.check_geometric(weight, max_err)
    with pytest.raises(ValueError):
        api.geometric_pass(np.zeros((3, 16, 16), f32), [np.eye(3, 4)] * 3, SimpleNamespace(iterations=1), [0],
                           weight=weight, max_err=max_err)


@pytest.mark.parametrize("kw", [dict(refs=[3]), dict(refs=[]), dict(geo_iterations=-1), dict(geo_iterations=1.5),
                                dict(images=np.zeros((3, 16, 16, 3), f32)), dict(Ps=[np.eye(3, 4)] * 2), dict(max_views=0)])
def test_geometric_pass_refuses_bad_arguments_before_any_cuda_call(monkeypatch, kw):
    from gipuma_b200 import api

    def no_context(*a, **k):
        raise AssertionError("a context was created for arguments that must be refused")
    monkeypatch.setattr(api, "Context", no_context)
    args = dict(images=np.zeros((3, 16, 16), f32), Ps=[np.eye(3, 4)] * 3, params=SimpleNamespace(iterations=1), refs=[0])
    args.update(kw)
    with pytest.raises(ValueError):
        api.geometric_pass(**args)


def test_c_abi_refuses_null_contexts_and_arguments():
    from gipuma_b200 import api
    lib = api.load_library()
    depth = np.zeros((8, 8), f32)
    assert lib.gpm_set_geometric(None, ctypes.c_float(1.0), ctypes.c_float(1.0)) == -1
    assert lib.gpm_set_view_depth(None, 0, ctypes.c_void_p(depth.ctypes.data), 0, 0) == -1
    assert "null" in lib.gpm_last_error().decode()

"""The reprojection rule of the depth-map fusion (DESIGN.md §22) without a GPU: the C restatement on hand-made rigs with known
answers (each threshold on either side of its exact value, strict comparisons, a target point behind the reference camera,
NaN depths, disp_thresh unread, the same vertex as the disparity rule's), an exact change of the world's scale, the struct
layout, and the refusal of bad rules before any CUDA call."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

F, W, H, Z0 = 100.0, 40, 24, 10.0          # focal length, image size, plane depth
ARGS = dict(depth_min=1.0, depth_max=100.0, disp_thresh=0.1, normal_thresh=30.0)
LOOSE = dict(reproj_px=1e6, depth_rel=1e6)


def _P(c=(0.0, 0.0, 0.0)):
    """Camera with R = I at c, principal point at the image centre."""
    K = np.array([[F, 0, W / 2], [0, F, H / 2], [0, 0, 1.0]])
    return K @ np.hstack([np.eye(3), -np.array(c, dtype=np.float64)[:, None]])


def _plane(n_views, depths=None):
    """Every camera looks down +z at the plane z = Z0; view i's depth map holds depths[i] (default Z0)."""
    n4 = np.zeros((n_views, H, W, 4), np.float32)
    n4[..., 2] = -1.0
    n4[..., 3] = Z0
    for i, d in enumerate(depths or []):
        n4[i, ..., 3] = d
    return n4


# camera 1 sits 2 to the right: a plane point seen at column x in view 0 is at column x - 20 in view 1
SHIFT = 20
PS2 = [_P(), _P((2.0, 0.0, 0.0))]


def _fuse(n4, Ps, num_consistent=1, rule="reprojection", **kw):
    from gipuma_b200 import api
    from oracle import pyfusion_rule
    args = dict(ARGS, **{k: kw.pop(k) for k in list(kw) if k in ARGS})
    return pyfusion_rule.fuse(n4, api.fuse_cameras(Ps), num_consistent=num_consistent, rule=rule, **args, **kw)


def _pass0(delta, **rule):
    """Pass 0 of the wide-baseline rig with view 1's depths off by the factor 1 + delta: the number of vertices."""
    v, _, _ = _fuse(_plane(2, [Z0, Z0 * (1.0 + delta)]), PS2, refs=(0, 1), **rule)
    return len(v)


def test_the_disparity_rule_of_the_new_restatement_is_the_old_one():
    from gipuma_b200 import api
    from oracle import pyfusion
    rng = np.random.default_rng(3)
    n4 = _plane(3)
    n4[..., 3] *= rng.uniform(0.97, 1.03, size=(3, H, W)).astype(np.float32)
    Ps = PS2 + [_P((-0.5, 0.3, 0.0))]
    grey = rng.uniform(0, 255, size=(3, H, W)).astype(np.float32)
    a = pyfusion.fuse(n4, api.fuse_cameras(Ps), num_consistent=1, images=grey, **ARGS)
    b = _fuse(n4, Ps, rule="disparity", images=grey, reproj_px=-1.0, depth_rel=float("nan"))
    assert len(a[0]) > 0 and a[0].tobytes() == b[0].tobytes()
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_reproj_px_decides_on_either_side_of_the_parallax():
    """View 1's point is off by delta along its ray: it reprojects shift * delta / (1 + delta) pixels from the reference
    pixel, at the relative depth delta."""
    delta = 0.05
    e = SHIFT * delta / (1 + delta)                            # 0.952 px
    full = H * (W - SHIFT)
    assert _pass0(delta, reproj_px=e * 1.01, depth_rel=1e6) == full
    assert _pass0(delta, reproj_px=e * 0.99, depth_rel=1e6) == 0
    assert _pass0(delta, reproj_px=1e6, depth_rel=delta * 1.01) == full
    assert _pass0(delta, reproj_px=1e6, depth_rel=delta * 0.99) == 0
    # both must hold
    assert _pass0(delta, reproj_px=e * 1.01, depth_rel=delta * 0.99) == 0
    assert _pass0(delta, reproj_px=e * 0.99, depth_rel=delta * 1.01) == 0


def _reprojection_of(n4, Ps, x, y, j):
    """fp32 restatement in numpy, one round-to-nearest step per operation, of the reprojection rule's quantities for
    reference pixel (x, y) of view 0 and view j: (e, relative depth difference)."""
    from gipuma_b200 import api
    f32 = np.float32
    cams = api.fuse_cameras(Ps)

    def arr(c):
        return np.array(c.M_inv[:], np.float32).reshape(3, 3), np.array(c.P[:], np.float32).reshape(3, 4)

    def dot3(a, X):
        return (a[0] * X[0] + a[1] * X[1]) + a[2] * X[2]

    def backproject(c, u, v, d):
        Mi, P = arr(c)
        abc = (d * u - P[0, 3], d * v - P[1, 3], d - P[2, 3])
        return [dot3(Mi[k], abc) for k in range(3)]

    def project(c, X):
        P = arr(c)[1]
        return [dot3(P[k], X) + P[k, 3] for k in range(3)]

    dr = n4[0, y, x, 3]
    X = backproject(cams[0], f32(x), f32(y), dr)
    h = project(cams[j], X)
    u, v = np.floor(h[0] / h[2] + f32(0.5)), np.floor(h[1] / h[2] + f32(0.5))
    Xj = backproject(cams[j], u, v, n4[j, int(v), int(u), 3])
    g = project(cams[0], Xj)
    dx, dy = g[0] / g[2] - f32(x), g[1] / g[2] - f32(y)
    return np.sqrt(dx * dx + dy * dy), np.abs(g[2] - dr) / dr


def test_the_comparisons_are_strict():
    n4 = _plane(2, [Z0, Z0 * 1.05])
    n4[0, ..., 3] = 0.0
    n4[0, 7, 31, 3] = Z0                                       # one reference pixel
    e, rel = _reprojection_of(n4, PS2, 31, 7, 1)
    assert e > 0 and rel > 0
    up = lambda t: float(np.nextafter(t, np.float32(np.inf)))   # noqa: E731
    for rule, ok in ((dict(reproj_px=float(e), depth_rel=1e6), 0), (dict(reproj_px=up(e), depth_rel=1e6), 1),
                     (dict(reproj_px=1e6, depth_rel=float(rel)), 0), (dict(reproj_px=1e6, depth_rel=up(rel)), 1)):
        v, src, _ = _fuse(n4, PS2, refs=(0, 1), **rule)
        assert len(v) == ok, rule
        if ok:
            assert src.tolist() == [[0, 7 * W + 31]]


def test_a_target_point_behind_the_reference_camera_is_rejected():
    """View 1 sits 20 behind view 0: X on the plane is at depth 30 in view 1; its own depth d puts its point at z = d - 20 in
    view 0, behind the camera for d < 20 and on the camera's plane for d = 20, whatever the thresholds."""
    Ps = [_P(), _P((0.0, 0.0, -20.0))]
    for d, want in ((15.0, 0), (20.0, 0), (25.0, H * W)):
        v, _, _ = _fuse(_plane(2, [Z0, d]), Ps, refs=(0, 1), **LOOSE)
        assert len(v) == want, d


def test_nan_depths_are_never_consistent():
    n4 = _plane(2)
    n4[1, :, :10, 3] = np.nan                                  # the targets of view 0's columns 20..29
    v, src, used = _fuse(n4, PS2, refs=(0, 1), **LOOSE)
    assert len(v) == H * (W - SHIFT - 10) and (src[:, 1] % W >= 30).all()
    n4 = _plane(2)
    n4[0, :, 25:, 3] = np.nan                                  # references
    v, src, _ = _fuse(n4, PS2, refs=(0, 1), **LOOSE)
    assert len(v) == H * (25 - SHIFT) and (src[:, 1] % W < 25).all()


def test_disp_thresh_is_not_read():
    n4 = _plane(2, [Z0, Z0 * 1.05])
    want = _fuse(n4, PS2, reproj_px=1.0, depth_rel=0.06)
    assert len(want[0]) > 0
    for dt in (1e-9, 1e9, 0.0, -1.0, float("nan")):
        got = _fuse(n4, PS2, reproj_px=1.0, depth_rel=0.06, disp_thresh=dt)
        assert got[0].tobytes() == want[0].tobytes() and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])


def test_the_vertex_equals_the_disparity_rules_when_both_accept_the_same_views():
    Ps = PS2 + [_P((-1.0, 0.5, 0.0))]
    grey = np.random.default_rng(1).uniform(0, 255, size=(3, H, W)).astype(np.float32)
    a = _fuse(_plane(3), Ps, rule="disparity", images=grey)
    b = _fuse(_plane(3), Ps, images=grey)
    assert len(a[0]) > H * (W - SHIFT) and a[0].tobytes() == b[0].tobytes()
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_a_change_of_the_worlds_scale_changes_no_decision():
    """P's fourth column, the depths and the depth range times 2^-10: the same sources and masks, the vertices' positions
    times 2^-10 exactly, the same normals and colours.  Every operation of the rule is homogeneous in the scale."""
    rng = np.random.default_rng(11)
    Ps = [_P(), _P((2.0, 0.0, 0.0)), _P((-1.0, 0.7, 0.3)), _P((0.5, -1.5, -0.2))]
    n4 = _plane(4)
    n4[..., 3] *= rng.uniform(0.98, 1.02, size=(4, H, W)).astype(np.float32)
    n4[..., :3] += rng.normal(scale=0.2, size=(4, H, W, 3)).astype(np.float32)
    grey = rng.uniform(0, 255, size=(4, H, W)).astype(np.float32)
    s = 2.0 ** -10
    sPs = [np.hstack([P[:, :3], P[:, 3:] * s]) for P in Ps]
    sn4 = n4.copy()
    sn4[..., 3] *= np.float32(s)
    rule = dict(reproj_px=0.7, depth_rel=0.01, normal_thresh=20.0, images=grey)
    v, src, used = _fuse(n4, Ps, num_consistent=2, **rule)
    sv, ssrc, sused = _fuse(sn4, sPs, num_consistent=2, depth_min=s * 1.0, depth_max=s * 100.0, **rule)
    assert 0 < len(v) < 4 * H * W and np.array_equal(src, ssrc) and np.array_equal(used, sused)
    for k in ("x", "y", "z"):
        assert np.array_equal(sv[k], v[k] * np.float32(s))
    for k in ("nx", "ny", "nz", "red", "green", "blue"):
        assert np.array_equal(sv[k], v[k])
    # the disparity rule with the same disp_thresh does not keep its decisions
    d = _fuse(n4, Ps, num_consistent=2, rule="disparity", normal_thresh=20.0)
    sd = _fuse(sn4, sPs, num_consistent=2, rule="disparity", normal_thresh=20.0, depth_min=s * 1.0, depth_max=s * 100.0)
    assert not np.array_equal(d[1], sd[1])


def test_fusion_rule_layout_matches_ctypes(tmp_path):
    from gipuma_b200 import api
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gipuma_b200.h"\nint main(void){ printf("%zu %zu %zu %d %d\\n", '
                   'sizeof(gpm_fuse_rule), offsetof(gpm_fuse_rule, reproj_px), offsetof(gpm_fuse_rule, depth_rel), '
                   'GPM_FUSE_DISPARITY, GPM_FUSE_REPROJECTION); return 0; }\n')
    exe = str(tmp_path / "t")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(root, "include"), str(src), "-o", exe])
    got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(api.GpmFuseRule), api.GpmFuseRule.reproj_px.offset, api.GpmFuseRule.depth_rel.offset,
                   api.FUSE_RULES["disparity"], api.FUSE_RULES["reprojection"]]


def test_bad_rules_are_refused_before_any_cuda_call():
    from conftest import have_cuda
    from gipuma_b200 import api
    lib = api.load_library()
    n4 = _plane(2)
    P = np.ascontiguousarray(np.stack(PS2).reshape(-1))
    nan, inf = float("nan"), float("inf")

    def call(rule, **kw):
        d = api.GpmFuseDesc(2, W, H, n4.ctypes.data, None, 0, 0, P.ctypes.data_as(C.POINTER(C.c_double)), 1.0,
                            1.0, 100.0, 0.1, 30.0, 1, 0)
        for k, v in kw.items():
            setattr(d, k, v)
        r = api.GpmFuseResult(0, 0, None, None, None, 0.0, 0.0)
        return lib.gpm_fuse_with_rule(C.byref(d), None if rule is None else C.byref(api.GpmFuseRule(*rule)), C.byref(r)), \
            lib.gpm_last_error().decode()

    bad = [((-1, 2.0, 0.01), {}, "unknown rule kind"), ((2, 2.0, 0.01), {}, "unknown rule kind")]
    bad += [((1, t, 0.01), {}, "reproj_px must be finite and > 0") for t in (0.0, -1.0, nan, inf, -inf)]
    bad += [((1, 2.0, t), {}, "depth_rel must be finite and > 0") for t in (0.0, -1.0, nan, inf, -inf)]
    # what gpm_fuse refuses is still refused, under either rule
    for rule in (None, (0, 0.0, 0.0), (1, 2.0, 0.01)):
        bad += [(rule, kw, msg) for kw, msg in ((dict(n_views=1), "n_views"), (dict(P=None), "norm4 and P are required"),
                                                (dict(num_consistent=0), "num_consistent"), (dict(normal_thresh=0.0), "normal_thresh"),
                                                (dict(depth_max=0.5), "depth_min"), (dict(width=0), "bad image size"),
                                                (dict(images=n4.ctypes.data, channels=3), "channels"),
                                                (dict(cam_scale=0.0), "bad projection matrix"))]
    bad += [(rule, dict(disp_thresh=0.0), "disp_thresh") for rule in (None, (0, 2.0, 0.01))]
    for rule, kw, msg in bad:
        rc, got = call(rule, **kw)
        assert rc == -1 and got.startswith("gpm_fuse: ") and msg in got, (rule, kw, rc, got)
    if not have_cuda():
        # valid descriptors, disp_thresh included under the reprojection rule where it is not read: they need a device
        for rule, kw in (((1, 2.0, 0.01), dict(disp_thresh=0.0)), ((1, 2.0, 0.01), dict(disp_thresh=nan)), ((0, -1.0, nan), {})):
            rc, got = call(rule, **kw)
            assert rc == -2, (rule, kw, got)


def test_api_refuses_bad_rules_before_the_library_loads(monkeypatch, tmp_path):
    from gipuma_b200 import api

    def boom():
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(api, "load_library", boom)
    n4 = _plane(2)
    nan = float("nan")
    cases = [(dict(rule="colmap"), "rule must be one of"), (dict(rule=None), "rule must be one of"),
             (dict(rule="disparity", reproj_px=2.0), "apply to rule='reprojection' only"),
             (dict(depth_rel=0.01), "apply to rule='reprojection' only")]
    cases += [(dict(rule="reprojection", reproj_px=t), "reproj_px must be finite and > 0") for t in (0.0, -2.0, nan, float("inf"), 1e39)]
    cases += [(dict(rule="reprojection", depth_rel=t), "depth_rel must be finite and > 0") for t in (0.0, -0.1, nan, 1e-50)]
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg.replace("(", r"\(")):
            api.fuse(n4, PS2, 1.0, 100.0, **kw)
        with pytest.raises(ValueError, match=msg.replace("(", r"\(")):
            api.fuse_batch_dir(str(tmp_path), [0, 1], PS2, 1.0, 100.0, **kw)
    assert api.FUSE_REPROJ_DEFAULTS == {"reproj_px": 2.0, "depth_rel": 0.01}

"""Depth-map fusion on the GPU (gpm_fuse_with_rule, DESIGN.md §12, §22) where it can go wrong: image sizes that leave the
last block of k_fuse_pixels, k_scan_blocks and k_compact partial, 2 to 256 views (the camera table at its full size),
inputs one ULP either side of every threshold, non-finite and degenerate inputs, and result buffers too small for the
cloud.  Every run equals the C restatement (oracle/fusion_rule_oracle.c) bit for bit under both rules, and every
threshold case checks that its inputs produce both outcomes.  The first pass is also checked against the float64
reference (oracle/pyrecon64.py)."""
import ctypes as C

import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu

RULES = {"disparity": dict(disp_thresh=0.1), "reprojection": dict(reproj_px=1.0, depth_rel=0.01)}
F, CX, CY = 64.0, 8.0, 4.0                     # dyadic camera: every back-projection and projection of the rigs is exact


def _P(C0, f=F, cx=CX, cy=CY):
    K = np.array([[f, 0, cx], [0, f, cy], [0, 0, 1.0]])
    return K @ np.hstack([np.eye(3), -np.asarray(C0, np.float64)[:, None]])


def _args(rule, prm):
    a = dict(RULES[rule])
    a.update(prm)
    return a


def _fuse(n4, Ps, rule, images=None, threads=32, **prm):
    """The GPU and the restatement on one input: equal bit for bit.  Returns (vertices, info) of the GPU."""
    from gipuma_b200 import api
    from oracle import pyfusion_rule
    a = _args(rule, prm)
    kw = {} if rule == "disparity" else dict(reproj_px=a.pop("reproj_px"), depth_rel=a.pop("depth_rel"))
    v, info = api.fuse(n4, Ps, images=images, rule=rule, **a, **kw)
    ov, osrc, oused = pyfusion_rule.fuse(n4, api.fuse_cameras(Ps), images=images, threads=threads, rule=rule,
                                         **dict(dict(disp_thresh=0.1), **a), **kw)
    assert len(v) == len(ov) == info["count"]
    assert np.array_equal(info["source"], osrc)
    # the float fields bit for bit, NaN equal to NaN (the GPU's NaN is 0x7fffffff, the host's keeps the sign and payload
    # of the NaN it came from); the colours byte for byte
    for k in ("x", "y", "z", "nx", "ny", "nz"):
        assert bits_equal(v[k], ov[k]) == 0, k
    for k in ("red", "green", "blue"):
        assert np.array_equal(v[k], ov[k]), k
    assert np.array_equal(info["used"], oused)
    return v, info


def _fused0(info, H, W):
    """Pass 0's fused pixels of view 0 as an [H, W] mask."""
    m = np.zeros(H * W, bool)
    m[info["source"][info["source"][:, 0] == 0, 1]] = True
    return m.reshape(H, W)


def _straddles(outcome):
    outcome = np.asarray(outcome, bool)
    assert outcome.any() and not outcome.all(), "the ladder does not straddle the edge: %s" % outcome.astype(int)


def _ladder(x0, k=6, step=1):
    """2k + 1 floats centred on float32(x0), `step` ULPs apart (consecutive floats by default)."""
    x0 = np.float32(x0)
    up, dn = [x0], [x0]
    for _ in range(k * step):
        up.append(np.nextafter(up[-1], np.float32(np.inf)))
        dn.append(np.nextafter(dn[-1], np.float32(-np.inf)))
    up, dn = up[::step], dn[::step]
    return np.array(dn[:0:-1] + up, np.float32)


def _rendered(n_views, rows, cols, seed=3):
    from gipuma_b200 import scene as S
    fx = 1.2 * max(rows, cols)
    K = np.array([[fx, 0, cols / 2], [0, fx, rows / 2], [0, 0, 1.0]])
    Ps = S.synthetic_rig(n_views - 1, K, 500.0, 5.0, 25.0, seed=seed)
    hf = S.HeightField(z0=500.0, unit=500.0 / fx, seed=9)
    return S.render_norm4(Ps, 1.0, rows, cols, hf), Ps


RENDER = dict(depth_min=300.0, depth_max=800.0, normal_thresh=30.0)


@pytest.mark.parametrize("rule", list(RULES))
@pytest.mark.parametrize("size", [(1, 1), (7, 5), (41, 23), (255, 1), (1, 257), (129, 97)])
def test_gpu_fusion_at_ragged_sizes(size, rule):
    """Sizes that are not whole blocks of 256 (and 1 x 1): the restatement bit for bit, grey and RGBA, and pass 0 against
    float64 where its decisions are certain."""
    from gipuma_b200 import api
    from oracle import pyrecon64
    W, H = size
    n4, Ps = _rendered(5, H, W)
    rng = np.random.default_rng(W * 1000 + H)
    grey = rng.integers(0, 256, (5, H, W)).astype(np.float32)
    rgba = rng.uniform(-10, 265, (5, H, W, 4)).astype(np.float32)
    for images in (None, grey, rgba):
        v, info = _fuse(n4, Ps, rule, images=images, num_consistent=1, **RENDER)
        ref = pyrecon64.first_pass(n4, api.fuse_cameras(Ps), num_consistent=1, images=images, rule=rule,
                                   **dict(RENDER, **RULES[rule]))
        pyrecon64.check_first_pass(ref, v, info["source"], W, images=images is not None)
    if min(W, H) > 1:
        assert len(v) > 0.2 * W * H and ref["certain"].mean() > 0.9


def test_gpu_fusion_at_a_ragged_dtu_size():
    """49 DTU cameras at 1601 x 1201: a partial last block and more than 1024 blocks for the scan.  The first two passes
    equal the restatement exactly; on a seeded sample of later passes every vertex is the restatement's candidate of its
    pixel, and every candidate not emitted was marked by an earlier pass."""
    from gipuma_b200 import api, scene as S
    from oracle import pyfusion_rule
    Ps = [S.load_dtu_projections()[i] for i in range(49)]
    H, W = 1201, 1601
    hf = S.HeightField(z0=550.0, unit=550.0 / S.prepare_cameras(Ps[:1])[0].fx, seed=77)
    gt = S.render_norm4(Ps, 1.0, H, W, hf)
    prm = dict(depth_min=300.0, depth_max=800.0, disp_thresh=0.1, normal_thresh=30.0, num_consistent=3)
    v, info = api.fuse(gt, Ps, **prm)
    cams = api.fuse_cameras(Ps)
    src = info["source"]
    ov, osrc, _ = pyfusion_rule.fuse(gt, cams, refs=(0, 2), threads=32, **prm)
    k = int((src[:, 0] < 2).sum())
    assert k == len(ov) > 0 and np.array_equal(src[:k], osrc) and v[:k].tobytes() == ov.tobytes()
    for r in np.random.default_rng(2027).choice(np.arange(2, 49), 3, replace=False):
        cv, csrc, _ = pyfusion_rule.fuse(gt, cams, refs=(int(r), int(r) + 1), threads=32, **prm)
        mine = src[:, 0] == r
        pos = np.searchsorted(csrc[:, 1], src[mine, 1])
        assert (pos < len(csrc)).all() and np.array_equal(csrc[pos, 1], src[mine, 1])
        assert v[mine].tobytes() == cv[pos].tobytes()
        missed = np.setdiff1d(csrc[:, 1], src[mine, 1])
        assert info["used"][r].reshape(-1)[missed].all()


@pytest.mark.parametrize("rule", list(RULES))
@pytest.mark.parametrize("n", [2, 3, 33, 255, 256])
def test_gpu_fusion_view_counts(n, rule):
    """2 to 256 views (256 fills the shared camera table, 22.5 KB) at 61 x 45, with num_consistent 1, n - 1 and n; n
    asks for more views than there are others, so nothing fuses and nothing is marked."""
    n4, Ps = _rendered(n, 45, 61)
    for nc in sorted({1, n - 1, n}):
        v, info = _fuse(n4, Ps, rule, num_consistent=nc, **RENDER)
        if nc == 1:
            assert len(v) > 100
        if nc == n:
            assert len(v) == 0 and not info["used"].any()


# ---- thresholds: an exact rig, and ladders of consecutive floats across each edge ----

W_E, H_E, Z = 24, 13, 32.0


def _two_view(rule, ref_depth, tgt_depth, b=(0.5, 0.0, 0.0), ref_normal=(0.0, 0.0, -1.0), tgt_normal=None, **prm):
    """View 0 at the origin, view 1 at b, both R = I: a pixel (x, y) at depth Z lands on (x - 64 b_x / Z, y - 64 b_y / Z)
    of view 1.  Depths and normals: scalars, or [H, W] / [H, W, 3] maps.  Returns (fused [H, W] of pass 0, info)."""
    n4 = np.zeros((2, H_E, W_E, 4), np.float32)
    n4[0, ..., 3], n4[1, ..., 3] = ref_depth, tgt_depth
    n4[0, ..., :3] = ref_normal
    n4[1, ..., :3] = ref_normal if tgt_normal is None else tgt_normal
    a = dict(depth_min=1.0, depth_max=100.0, normal_thresh=30.0, num_consistent=1)
    a.update(prm)
    _, info = _fuse(n4, [_P((0, 0, 0)), _P(b)], rule, threads=4, **a)
    return _fused0(info, H_E, W_E), info


def _row_ladder(base, values, row=0, col=4):
    m = np.full((H_E, W_E), np.float32(base), np.float32)
    m[row, col:col + len(values)] = values
    return m


@pytest.mark.parametrize("rule", list(RULES))
@pytest.mark.parametrize("edge", ["min", "max"])
def test_gpu_fusion_depth_range_edges(rule, edge):
    """The reference depth and the target depth on depth_min / depth_max and one ULP either side."""
    lad = _ladder(Z)
    lim = dict(depth_min=Z, depth_max=100.0) if edge == "min" else dict(depth_min=1.0, depth_max=Z)
    inside = np.float32(Z + 0.25 if edge == "min" else Z - 0.25)       # within the reprojection rule's depth_rel
    # the reference's depth: a pixel whose own depth is out of range never fuses
    fused, _ = _two_view(rule, _row_ladder(inside, lad), inside, **lim)
    _straddles(fused[0, 4:4 + len(lad)])
    assert np.array_equal(fused[0, 4:4 + len(lad)], (lad >= Z) if edge == "min" else (lad <= Z))
    # the target's depth: view 0's pixel x sees view 1's pixel x - 1
    fused, _ = _two_view(rule, inside, _row_ladder(inside, lad, col=3), **lim)
    _straddles(fused[0, 4:4 + len(lad)])


def test_gpu_fusion_disparity_edge():
    """|f 0.54 / z - f 0.54 / d_j| against disp_thresh: the target depth laddered across the analytic crossing."""
    fb = np.float64(np.float32(np.float32(F) * np.float32(0.54)))
    for thr in (0.1, 0.02):
        t = np.float32(thr)
        for cross in (fb / (fb / Z - t), fb / (fb / Z + t)):
            lad = _ladder(cross, 8)
            fused, _ = _two_view("disparity", Z, _row_ladder(Z, lad, col=3), disp_thresh=thr)
            _straddles(fused[0, 4:4 + len(lad)])


def test_gpu_fusion_reprojection_distance_edge():
    """A target depth of 16 against a reference depth of 32, cameras 1 apart: the target's point reprojects exactly 2
    pixels away, on reproj_px = 2; the ladder puts it on both sides."""
    lad = _ladder(16.0)
    fused, _ = _two_view("reprojection", Z, _row_ladder(Z, lad, col=2), b=(1.0, 0.0, 0.0), reproj_px=2.0, depth_rel=1.0)
    _straddles(fused[0, 4:4 + len(lad)])


def test_gpu_fusion_relative_depth_edge():
    """|z_j - d| / d against depth_rel = 0.25 with d = 32: exactly on the edge at target depths 40 and 24."""
    for cross in (40.0, 24.0):
        lad = _ladder(cross)
        fused, _ = _two_view("reprojection", Z, _row_ladder(Z, lad, col=3), reproj_px=4.0, depth_rel=0.25)
        _straddles(fused[0, 4:4 + len(lad)])
        assert np.array_equal(fused[0, 4:4 + len(lad)], np.abs(lad.astype(np.float64) - Z) / Z < 0.25)


@pytest.mark.parametrize("rule", list(RULES))
@pytest.mark.parametrize("deg", [30.0, 90.0, 180.0])
def test_gpu_fusion_normal_edge(rule, deg):
    """The dot product of the normals against cos(normal_thresh), laddered across it; at 90 degrees a perpendicular
    normal (dot exactly 0) as well."""
    import math
    c = np.float32(math.cos(float(np.float32(deg)) * math.pi / 180.0))
    lad = _ladder(c)
    tn = np.zeros((H_E, W_E, 3), np.float32)
    tn[..., 2] = -1.0
    tn[0, 3:3 + len(lad), 2] = -lad                            # dot with (0, 0, -1) is exactly the ladder value
    if deg == 90.0:
        tn[1, 3] = (1.0, 0.0, 0.0)
    fused, _ = _two_view(rule, Z, Z, tgt_normal=tn, normal_thresh=deg)
    _straddles(fused[0, 4:4 + len(lad)])
    assert np.array_equal(fused[0, 4:4 + len(lad)], lad > c)
    if deg == 90.0:
        assert not fused[1, 4]


@pytest.mark.parametrize("rule", list(RULES))
@pytest.mark.parametrize("axis,sign", [(0, 1), (0, -1), (1, 1), (1, -1)])
def test_gpu_fusion_image_border_edges(rule, axis, sign):
    """Cameras a quarter apart: at depth 32 every projection lands on a half pixel, so the first column (row) lands on
    u = -0.5 and the last on W - 0.5.  The reference depth is laddered across 32 along the other axis, 32 ULPs apart: the
    back-projection d x rounds at a coarser step than d's own ULP, so consecutive depths would all land on the tie."""
    b = [0.0, 0.0, 0.0]
    b[axis] = 0.25 * sign
    n = H_E if axis == 0 else W_E
    lad = _ladder(Z, n // 2, step=32)[:n]
    dep = np.empty((H_E, W_E), np.float32)
    if axis == 0:
        dep[:] = lad[:H_E, None]
    else:
        dep[:] = lad[None, :W_E]
    fused, _ = _two_view(rule, dep, Z, b=tuple(b))
    edge = 0 if sign > 0 else (W_E if axis == 0 else H_E) - 1
    probe = fused[:, edge] if axis == 0 else fused[edge, :]
    _straddles(probe)


@pytest.mark.parametrize("rule", list(RULES))
def test_gpu_fusion_target_camera_plane_edge(rule):
    """The reference point (0, 0, 32) against target cameras at (0, 0, c), c laddered across 32: on the target's z = 0
    plane (c = 32) and behind it nothing is consistent; in front, the target pixel at the principal point holds the
    exact depth 32 - c."""
    lad = _ladder(Z, 4)
    n = 1 + len(lad)
    n4 = np.zeros((n, H_E, W_E, 4), np.float32)
    n4[..., :3] = (0.0, 0.0, -1.0)
    n4[0, int(CY), int(CX), 3] = Z
    for k, c in enumerate(lad):
        n4[1 + k, int(CY), int(CX), 3] = max(np.float32(Z) - c, np.float32(0.0))
    Ps = [_P((0, 0, 0))] + [_P((0.0, 0.0, float(c))) for c in lad]
    _, info = _fuse(n4, Ps, rule, threads=4, depth_min=2.0 ** -30, depth_max=100.0, normal_thresh=30.0, num_consistent=1)
    marked = info["used"][1:, int(CY), int(CX)].astype(bool)
    _straddles(marked)
    assert np.array_equal(marked, lad < np.float32(Z))


SPECIALS = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1e-40, -1e-40, 1e-45], np.float32)


@pytest.mark.parametrize("rule", list(RULES))
def test_gpu_fusion_non_finite_inputs(rule):
    """NaN, +-inf, -0 and subnormal depths and normal components, and colours that are NaN, negative or above 255."""
    n4, Ps = _rendered(5, 23, 41)
    rng = np.random.default_rng(17)
    for ch in range(4):
        hit = rng.random(n4.shape[:3]) < 0.08
        n4[..., ch][hit] = rng.choice(SPECIALS, int(hit.sum()))
    rgba = rng.uniform(0, 255, n4.shape).astype(np.float32)
    hit = rng.random(rgba.shape) < 0.1
    rgba[hit] = rng.choice(np.array([np.nan, -7.0, 300.0, np.inf, -np.inf], np.float32), int(hit.sum()))
    for images in (None, np.ascontiguousarray(rgba[..., 0]), rgba):
        v, info = _fuse(n4, Ps, rule, images=images, num_consistent=1, **RENDER)
        assert len(v) > 50


@pytest.mark.parametrize("rule", list(RULES))
def test_gpu_fusion_degenerate_normal_sums_and_half_colours(rule):
    """Two targets whose normals cancel the reference's (the len > 0 branch: a zero normal), and colours whose mean is
    exactly k + 0.5 (rounded half up), NaN (0), negative (0) or above 255 (255)."""
    n4 = np.zeros((3, H_E, W_E, 4), np.float32)
    n4[..., 3] = Z
    n4[0, ..., :3] = (0.0, 0.0, -1.0)
    n4[1, ..., :3] = (0.0, 0.875, 0.5)
    n4[2, ..., :3] = (0.0, -0.875, 0.5)
    rgba = np.zeros((3, H_E, W_E, 4), np.float32)
    rgba[0, ..., :3] = (100.0, np.nan, -30.0)
    rgba[1, ..., :3] = (101.0, 5.0, 10.0)
    rgba[2, ..., :3] = (103.0, 5.0, 8.0)                         # red: 304 / 3 -> 101.33
    rgba[0, 0, :, 0] = 600.0                                   # (600 + 101 + 103) / 3 > 255
    rgba[0, 1, :, 0] = 0.5                                     # (0.5 + 101 + 103) / 3 = 68.1666
    rgba[1, 2, :, 0], rgba[2, 2, :, 0], rgba[0, 2, :, 0] = 1.0, 2.0, 1.5     # mean 1.5 -> 2
    Ps = [_P((0, 0, 0)), _P((0.5, 0, 0)), _P((-0.5, 0, 0))]
    v, info = _fuse(n4, Ps, rule, images=rgba, threads=4, depth_min=1.0, depth_max=100.0, normal_thresh=180.0,
                    num_consistent=2)
    first = info["source"][:, 0] == 0
    assert first.sum() > 50
    assert (v["nx"][first] == 0).all() and (v["ny"][first] == 0).all() and (v["nz"][first] == 0).all()
    assert (v["green"][first] == 0).all() and (v["blue"][first] == 0).all()
    rows = info["source"][first, 1] // W_E
    assert (v["red"][first][rows == 0] == 255).all() and (v["red"][first][rows == 2] == 2).all()
    # two views, grey: every vertex is the mean of 100 and 103, 101.5 -> 102
    g = np.stack([np.full((H_E, W_E), 100.0, np.float32), np.full((H_E, W_E), 103.0, np.float32)])
    n2 = np.zeros((2, H_E, W_E, 4), np.float32)
    n2[..., :3], n2[..., 3] = (0.0, 0.0, -1.0), Z
    v2, _ = _fuse(n2, Ps[:2], rule, images=g, threads=4, depth_min=1.0, depth_max=100.0, normal_thresh=30.0, num_consistent=1)
    assert len(v2) > 50 and (v2["red"] == 102).all() and (v2["blue"] == 102).all()


# ---- result buffers smaller than the cloud ----

@pytest.fixture(scope="module")
def cap_case():
    from gipuma_b200 import api
    n4, Ps = _rendered(5, 23, 41, seed=5)
    v, info = api.fuse(n4, Ps, num_consistent=1, **RENDER)
    assert len(v) > 100 and len(np.unique(info["source"][:, 0])) >= 3
    return n4, Ps, v, info


def _raw_fuse(n4, Ps, cap, vertices=True, source=True, used=True):
    """gpm_fuse_with_rule through ctypes with `cap` records; the buffers are filled with 0xAB beforehand."""
    from gipuma_b200 import api
    lib = api.load_library()
    n, H, W = n4.shape[:3]
    P = np.ascontiguousarray(np.stack(Ps).reshape(-1), np.float64)
    d = api.GpmFuseDesc(n, W, H, n4.ctypes.data, None, 0, 0, P.ctypes.data_as(C.POINTER(C.c_double)), 1.0,
                        RENDER["depth_min"], RENDER["depth_max"], 0.1, RENDER["normal_thresh"], 1, 0)
    rule = api.GpmFuseRule(0, 0.0, 0.0)
    vb = np.full(max(cap, 1) * 27 + 64, 0xAB, np.uint8) if vertices else None
    sb = np.full((max(cap, 1) + 8, 2), -0x54545455, np.int32) if source else None
    ub = np.full((n, H, W), 0xAB, np.uint8) if used else None
    r = api.GpmFuseResult(0, cap, None if vb is None else vb.ctypes.data, None if sb is None else sb.ctypes.data,
                          None if ub is None else ub.ctypes.data, 0.0, 0.0)
    rc = lib.gpm_fuse_with_rule(C.byref(d), C.byref(rule), C.byref(r))
    return rc, int(r.count), vb, sb, ub, lib.gpm_last_error().decode()


def test_gpu_fusion_capacity_is_a_prefix(cap_case):
    """Capacity 0 with no buffers counts; any capacity below the count returns -1 with the full count, fills exactly the
    fitting prefix of the full run (inside a pass or on a pass boundary) and leaves the rest untouched, with complete
    used masks; each of the buffers may be left out."""
    n4, Ps, v, info = cap_case
    cnt, src, used = info["count"], info["source"], info["used"]
    full = v.tobytes()
    rc, count, *_ = _raw_fuse(n4, Ps, 0, vertices=False, source=False, used=False)
    assert rc == -1 and count == cnt
    starts = [int(np.argmax(src[:, 0] == r)) for r in np.unique(src[:, 0])[1:]]
    caps = sorted(c for c in {cnt - 1, 1} | {s + d for s in starts for d in (-1, 0, 1)} if 1 <= c < cnt)
    for cap in caps:
        for vert, sour, us in ((True, True, True), (True, False, True), (False, True, True), (True, True, False)):
            rc, count, vb, sb, ub, msg = _raw_fuse(n4, Ps, cap, vert, sour, us)
            assert rc == -1 and count == cnt and "capacity" in msg, (cap, rc, count, msg)
            if vert:
                assert vb[:27 * cap].tobytes() == full[:27 * cap] and (vb[27 * cap:] == 0xAB).all(), cap
            if sour:
                assert np.array_equal(sb[:cap], src[:cap]) and (sb[cap:] == -0x54545455).all(), cap
            if us:
                assert np.array_equal(ub, used), cap
    rc, count, vb, sb, ub, _ = _raw_fuse(n4, Ps, cnt)
    assert rc == 0 and count == cnt and vb[:27 * cnt].tobytes() == full and np.array_equal(sb[:cnt], src)

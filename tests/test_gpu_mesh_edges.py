"""The meshing on the GPU (gpm_tsdf_integrate, gpm_mesh_extract; DESIGN.md §24) where it can go wrong: image sizes from
1 x 1, 1 to 256 views, voxels one ULP either side of every decision of the integration, exact result capacities, a box
whose D passes 2^31 bytes, a closed sphere at a size the CPU tests do not reach, and non-contiguous CUDA inputs.
Integrations equal the C restatement (oracle/mesh_oracle.c) bit for bit and the float64 reference (oracle/pyrecon64.py)
wherever its decisions are certain; every edge case checks that its inputs produce both outcomes."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DMIN, DMAX = 300.0, 800.0


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _tsdf(depth, Ps, origin, voxel, dims, trunc, dmin=DMIN, dmax=DMAX, threads=32):
    """The GPU and the restatement on one input, equal bit for bit; the GPU against float64 where certain.  Returns
    (D, Wt, share of certain voxels)."""
    from gipuma_b200 import api
    from oracle import pymesh, pyrecon64
    depth = np.ascontiguousarray(depth, np.float32)
    D, Wt, _ = api.tsdf_integrate(depth, Ps, origin, voxel, dims, trunc, dmin, dmax)
    cams = api.fuse_cameras(Ps)
    oD, oW = pymesh.tsdf(depth, cams, origin, voxel, dims, trunc, dmin, dmax, threads=threads)
    assert _bits_equal(D, oD) and _bits_equal(Wt, oW)
    certain = pyrecon64.check_tsdf(pyrecon64.tsdf(depth, cams, origin, voxel, dims, trunc, dmin, dmax), D, Wt)
    return D, Wt, certain / float(np.prod(dims))


def _rendered(n_views, rows, cols, seed=3):
    from gipuma_b200 import scene as S
    fx = 1.2 * max(rows, cols)
    K = np.array([[fx, 0, cols / 2], [0, fx, rows / 2], [0, 0, 1.0]])
    Ps = S.synthetic_rig(n_views - 1, K, 500.0, 5.0, 25.0, seed=seed)
    hf = S.HeightField(z0=500.0, unit=500.0 / fx, seed=9)
    n4 = S.render_norm4(Ps, 1.0, rows, cols, hf)
    return np.ascontiguousarray(n4[..., 3]), Ps


def _box_of(Ps, n=24):
    """A box around the surface point seen at the reference's centre: 70 x 70 x 40 world units in n^3 voxels."""
    voxel = float(np.float32(70.0 / n))
    return (-35.0, -35.0, 480.0), voxel, (n, n, n)


@pytest.mark.parametrize("size", [(1, 1), (7, 5), (129, 97)])
def test_gpu_tsdf_at_ragged_image_sizes(size):
    W, H = size
    dep, Ps = _rendered(5, H, W)
    origin, voxel, dims = _box_of(Ps)
    D, Wt, certain = _tsdf(dep, Ps, origin, voxel, dims, 3 * voxel)
    assert certain > 0.99
    if W * H > 1:
        assert (Wt > 0).any()


@pytest.mark.parametrize("n", [1, 2, 255, 256])
def test_gpu_tsdf_view_counts(n):
    """1 to 256 views at 61 x 45; voxels near the surface at the centre are seen by every view, so Wt reaches n.  A voxel
    is certain when all n of its projections are, so the certain share falls with n (98 % at 255 views)."""
    dep, Ps = _rendered(n, 45, 61)
    origin, voxel, dims = _box_of(Ps, 20)
    D, Wt, certain = _tsdf(dep, Ps, origin, voxel, dims, 3 * voxel)
    assert int(Wt.max()) == n and certain > 0.95


# ---- decisions of the integration on an exact rig: R = I, dyadic camera, voxel centres on its axis ----

F, CX, CY, W_E, H_E = 64.0, 8.0, 4.0, 16, 8


def _P(C0):
    K = np.array([[F, 0, CX], [0, F, CY], [0, 0, 1.0]])
    return K @ np.hstack([np.eye(3), -np.asarray(C0, np.float64)[:, None]])


def _ladder(x0, k=6):
    x0 = np.float32(x0)
    up, dn = [x0], [x0]
    for _ in range(k):
        up.append(np.nextafter(up[-1], np.float32(np.inf)))
        dn.append(np.nextafter(dn[-1], np.float32(-np.inf)))
    return np.array(dn[:0:-1] + up, np.float32)


def _straddles(outcome):
    outcome = np.asarray(outcome, bool)
    assert outcome.any() and not outcome.all(), "the ladder does not straddle the edge: %s" % outcome.astype(int)


def _axis_column(oz, nz, depth, trunc, dmin=1.0, dmax=1000.0, n=1, Ps=None):
    """A 2 x 2 x nz box of unit voxels whose first column of centres is (0, 0, oz + k + 0.5), on the optical axis of
    camera 0: it projects onto the principal point (8, 4), whose depth is `depth` (one per view with n views)."""
    dep = np.full((n, H_E, W_E), np.float32(1.0), np.float32)
    dep[:, int(CY), int(CX)] = depth
    Ps = Ps or [_P((0, 0, 0))] * n
    D, Wt, _ = _tsdf(dep, Ps, (-0.5, -0.5, float(oz)), 1.0, (2, 2, nz), trunc, dmin, dmax, threads=4)
    return D[:, 0, 0], Wt[:, 0, 0]


def test_gpu_tsdf_behind_the_truncation_edge():
    """sdf = d - z against -trunc: d = 50, trunc = 2, the voxel centre z laddered across 52 through the box's origin.
    Centres up to z = 47 are clamped to sdf = trunc (D = 1)."""
    seen = []
    for oz in _ladder(40.5):
        D, Wt = _axis_column(oz, 16, 50.0, 2.0)
        seen.append(Wt[11] > 0)
        assert (Wt[:7] == 1).all() and (D[:7] == 1.0).all()
    _straddles(seen)


def test_gpu_tsdf_depth_range_edges():
    """d on depth_min / depth_max and one ULP either side, one view per ladder value."""
    lad = _ladder(50.0)
    for lim in (dict(dmin=50.0, dmax=1000.0), dict(dmin=1.0, dmax=50.0)):
        _, Wt = _axis_column(48.5, 4, lad, 4.0, n=len(lad), **lim)
        assert Wt[0] == int(((lad >= lim["dmin"]) & (lad <= lim["dmax"])).sum())
        assert 0 < Wt[0] < len(lad)
        _straddles((lad >= lim["dmin"]) & (lad <= lim["dmax"]))


def test_gpu_tsdf_special_depths():
    """d = 0, -0, a subnormal, NaN and +-inf, one view each, around one valid view: only the valid view counts, and a
    subnormal depth is in range (depth_min 0) but far in front of the voxel."""
    d = np.array([50.0, 0.0, -0.0, 1e-40, np.nan, np.inf, -np.inf, 49.0], np.float32)
    D, Wt = _axis_column(48.5, 4, d, 4.0, dmin=0.0, dmax=100.0, n=len(d))
    assert Wt[0] == 2


def test_gpu_tsdf_at_a_camera_plane():
    """Voxel centres on and just behind camera 0's z = 0 plane (the origin laddered across -0.5): only centres in front
    take a sample."""
    seen = []
    for oz in _ladder(-0.5):
        _, Wt = _axis_column(oz, 2, 1.0, 4.0)
        seen.append(Wt[0] > 0)
    _straddles(seen)


def test_gpu_tsdf_on_pixel_borders():
    """Voxel centres at x = -8.5 .. 8.5, z = 64 project onto u = -0.5 .. 16.5, every one a half pixel: u = -0.5 is in
    the image, u = W - 0.5 is not."""
    dep = np.full((1, H_E, W_E), np.float32(64.5), np.float32)
    D, Wt, _ = _tsdf(dep, [_P((0, 0, 0))], (-9.0, -0.5, 63.5), 1.0, (18, 2, 2), 4.0, 1.0, 1000.0, threads=4)
    row = Wt[0, 0]
    assert row[0] == 1 and row[16] == 0
    _straddles(row)


# ---- extraction ----

def _raw_extract(D, Wt, vcap, fcap, mw=1):
    from gipuma_b200 import api
    lib = api.load_library()
    nz, ny, nx = D.shape
    d = api.GpmMeshDesc(D.ctypes.data, Wt.ctypes.data, 0, (C.c_float * 3)(0, 0, 0), 1.0, (C.c_int * 3)(nx, ny, nz), mw, 0)
    v = np.full((max(vcap, 1) + 4, 3), np.float32(-7.0))
    f = np.full((max(fcap, 1) + 4, 3), -7, np.int32)
    r = api.GpmMeshResult(0, 0, vcap, fcap, v.ctypes.data, f.ctypes.data, 0.0, 0.0)
    rc = lib.gpm_mesh_extract(C.byref(d), C.byref(r))
    return rc, (r.n_vertices, r.n_faces), v, f


def test_gpu_mesh_exact_capacities():
    """Capacities equal to the counts succeed; one vertex or one face short fails after filling what fits."""
    from gipuma_b200 import api
    rng = np.random.default_rng(8)
    D = rng.standard_normal((9, 10, 11)).astype(np.float32)
    Wt = rng.integers(0, 3, D.shape).astype(np.uint16)
    v0, f0, _ = api.extract_mesh(D, Wt, (0, 0, 0), 1.0, 1)
    nv, nf = len(v0), len(f0)
    rc, counts, v, f = _raw_extract(D, Wt, nv, nf)
    assert rc == 0 and counts == (nv, nf) and _bits_equal(v[:nv], v0) and np.array_equal(f[:nf], f0)
    assert (v[nv:] == -7.0).all() and (f[nf:] == -7).all()
    for vc, fc in ((nv - 1, nf), (nv, nf - 1)):
        rc, counts, v, f = _raw_extract(D, Wt, vc, fc)
        assert rc == -1 and counts == (nv, nf)
        assert _bits_equal(v[:vc], v0[:vc]) and np.array_equal(f[:fc], f0[:fc])
        assert (v[vc:] == -7.0).all() and (f[fc:] == -7).all()


def test_gpu_mesh_of_a_box_past_2_to_the_31_bytes():
    """2048 x 2048 x 130 unit voxels (D is 2.2 GB, 2.1 M blocks per scan), a plane at z = 127.25 and a fixed pattern of
    invalid points: the whole box's mesh equals bit for bit, vertex ids included, the restatement's mesh of the slab of
    layers 125-128 (origin z = 125, exact in fp32: no other layer has a vertex)."""
    import torch
    from gipuma_b200 import api
    from oracle import pymesh
    free, _ = torch.cuda.mem_get_info()
    if free < 12 * 2 ** 30:          # D, Wt and the extraction's buffers: an estimate from their sizes, not measured
        pytest.skip("%.1f GB free on the device; the box needs about 12 GB" % (free / 2 ** 30))
    nx, ny, nz = 2048, 2048, 130
    z = torch.arange(nz, dtype=torch.float32, device="cuda") + 0.5
    D = (z - 127.25).view(nz, 1, 1).expand(nz, ny, nx).contiguous()
    k = torch.arange(nz, device="cuda", dtype=torch.int64).view(nz, 1, 1)
    j = torch.arange(ny, device="cuda", dtype=torch.int64).view(1, ny, 1)
    i = torch.arange(nx, device="cuda", dtype=torch.int64).view(1, 1, nx)
    Wt = ((i * 7 + j * 13 + k * 3) % 97 != 0).to(torch.uint16)
    assert D.numel() * 4 > 2 ** 31
    v, f, _ = api.extract_mesh(D, Wt, (0.0, 0.0, 0.0), 1.0, 1)
    sD, sW = D[125:129].cpu().numpy(), Wt[125:129].cpu().numpy()
    del D, Wt
    torch.cuda.empty_cache()
    ov, of = pymesh.extract(sD, sW, (0.0, 0.0, 125.0), 1.0, 1)
    assert len(f) > 4 * 10 ** 6
    assert _bits_equal(v, ov) and np.array_equal(f, of)


def test_gpu_mesh_of_a_large_sphere_is_closed_and_oriented():
    """A sphere of radius 90 in a (257, 263, 251) box: every directed edge once and its reverse once, Euler characteristic
    2, a positive volume close to the sphere's, and every vertex within the float64 bound of its edge point."""
    from gipuma_b200 import api
    from oracle import pyrecon64
    n = (257, 263, 251)
    o, s, c, r = (0.0, 0.0, 0.0), 1.0, (128.3, 131.1, 125.7), 90.0
    x, y, z = (np.float32(o[a]) + (np.arange(n[a], dtype=np.float32) + np.float32(0.5)) * np.float32(s) for a in range(3))
    Z, Y, X = np.meshgrid(z.astype(np.float64), y.astype(np.float64), x.astype(np.float64), indexing="ij")
    D = (np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r).astype(np.float32)
    del X, Y, Z
    v, f, _ = api.extract_mesh(D, np.ones(D.shape, np.uint16), o, s, 1)
    V = len(v)
    de = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).astype(np.int64)
    key = np.sort(de[:, 0] * V + de[:, 1])
    assert (np.diff(key) > 0).all()                           # each directed edge once
    assert np.array_equal(key, np.sort(de[:, 1] * V + de[:, 0]))    # and its reverse once
    assert V - len(de) // 2 + len(f) == 2
    a, b, cc = (v[f[:, k]].astype(np.float64) for k in range(3))
    vol = np.einsum("ij,ij->i", a, np.cross(b, cc)).sum() / 6.0
    assert 0.9 < vol / (4.0 / 3.0 * np.pi * r ** 3) < 1.0
    assert pyrecon64.check_mesh_vertices(D, o, s, v) == V


def test_gpu_extract_mesh_of_non_contiguous_cuda_views():
    """A y-sub-box and a z-strided view of CUDA volumes equal the host meshes of the same boxes made contiguous."""
    import torch
    from gipuma_b200 import api
    rng = np.random.default_rng(21)
    D = rng.standard_normal((40, 48, 56)).astype(np.float32)
    Wt = rng.integers(0, 3, D.shape).astype(np.uint16)
    dD, dW = torch.from_numpy(D).cuda(), torch.from_numpy(Wt.astype(np.int32)).to(torch.uint16).cuda()
    for sl in ((slice(None), slice(7, 31), slice(None)), (slice(None, None, 3), slice(None), slice(None))):
        gv, gf, _ = api.extract_mesh(dD[sl], dW[sl], (0.5, -1.0, 2.0), 0.75, 1)
        hv, hf, _ = api.extract_mesh(np.ascontiguousarray(D[sl]), np.ascontiguousarray(Wt[sl]), (0.5, -1.0, 2.0), 0.75, 1)
        assert len(hf) > 100 and _bits_equal(gv, hv) and np.array_equal(gf, hf)

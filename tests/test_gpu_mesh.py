"""The meshing on the GPU (gpm_tsdf_integrate, gpm_mesh_extract; DESIGN.md §24): equal bit for bit to the C restatement
(oracle/mesh_oracle.c) on ground-truth maps and on PatchMatch outputs, for host and device inputs and on repeated runs;
unchanged by a change of the world's scale by 2^-10; exact on adversarial volumes; at the DTU size; and within a voxel of
the surface."""
import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu

DMIN, DMAX = 300.0, 800.0
REFS = list(range(0, 16, 2))


def _box(Ps, scale, rows, cols, hf, n, pad=3):
    """A box of n^3 voxels around the ground truth the views see (cubic voxels, `pad` voxels of margin)."""
    from gipuma_b200 import scene as S
    g = S.gt_points(Ps, scale, rows, cols, hf, stride=4)
    lo, hi = g.min(axis=0).astype(np.float64), g.max(axis=0).astype(np.float64)
    voxel = float(np.float32((hi - lo).max() / (n - 2 * pad)))
    origin = tuple(float(np.float32(x)) for x in lo - pad * voxel)
    return origin, voxel


@pytest.fixture(scope="module")
def rig():
    """8 reference views of 16 DTU cameras at 128 x 96: PatchMatch outputs and ground-truth maps."""
    from gipuma_b200 import api, scene as S
    rows, cols = 96, 128
    Ps = [S.load_dtu_projections()[i] for i in range(16)]
    scale = 1600.0 / cols
    cams = S.prepare_cameras(Ps, scale)
    hf = S.HeightField(z0=550.0, unit=550.0 / cams[0].fx, seed=77)
    images = np.stack([S.render_view(c, rows, cols, hf)[0] for c in cams])
    p = S.AlgorithmParameters(box_hsize=11, box_vsize=11, iterations=3, n_best=3, cost_comb=S.COMB_BEST_N, gamma=10.0)
    p.depthMin, p.depthMax = DMIN, DMAX
    n4, _, _ = api.batch_run(images, Ps, p, REFS, cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
    fPs = [Ps[r] for r in REFS]
    gt = S.render_norm4(fPs, scale, rows, cols, hf)
    origin, voxel = _box(fPs, scale, rows, cols, hf, 48)
    return dict(fPs=fPs, scale=scale, hf=hf, rows=rows, cols=cols, maps={"pm": np.ascontiguousarray(n4[..., 3]),
                                                                         "gt": np.ascontiguousarray(gt[..., 3])},
                origin=origin, voxel=voxel, dims=(48, 44, 40))


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _oracle_tsdf(depth, Ps, scale, origin, voxel, dims, trunc, slices=None):
    from gipuma_b200 import api
    from oracle import pymesh
    return pymesh.tsdf(depth, api.fuse_cameras(Ps, scale), origin, voxel, dims, trunc, DMIN, DMAX, slices, threads=16)


@pytest.mark.parametrize("maps", ["gt", "pm"])
@pytest.mark.parametrize("trunc_vox", [2.0, 5.0])
def test_gpu_tsdf_and_mesh_equal_the_c_restatement(rig, maps, trunc_vox):
    import torch
    from gipuma_b200 import api
    from oracle import pymesh
    dep = rig["maps"][maps]
    trunc = trunc_vox * rig["voxel"]
    args = (rig["origin"], rig["voxel"], rig["dims"], trunc, DMIN, DMAX)
    D, Wt, info = api.tsdf_integrate(dep, rig["fPs"], *args, cam_scale=rig["scale"])
    oD, oW = _oracle_tsdf(dep, rig["fPs"], rig["scale"], rig["origin"], rig["voxel"], rig["dims"], trunc)
    assert _bits_equal(D, oD) and _bits_equal(Wt, oW)
    assert (Wt > 0).mean() > 0.05 and (D[Wt > 0] < 0).any()
    # device inputs and a second run: the same bits
    dD, dW, dinfo = api.tsdf_integrate(torch.from_numpy(dep).cuda(), rig["fPs"], *args, cam_scale=rig["scale"])
    assert dinfo["upload_ms"] == 0.0 and dD.is_cuda
    assert _bits_equal(dD.cpu().numpy(), D) and _bits_equal(dW.cpu().numpy(), Wt)
    D2, W2, _ = api.tsdf_integrate(dep, rig["fPs"], *args, cam_scale=rig["scale"])
    assert _bits_equal(D2, D) and _bits_equal(W2, Wt)
    for mw in (1, 2, 3):
        v, f, _ = api.extract_mesh(D, Wt, rig["origin"], rig["voxel"], mw)
        ov, of = pymesh.extract(D, Wt, rig["origin"], rig["voxel"], mw)
        assert len(f) > 100 and _bits_equal(v, ov) and np.array_equal(f, of)
        dv, df, _ = api.extract_mesh(dD, dW, rig["origin"], rig["voxel"], mw)
        assert _bits_equal(dv, v) and np.array_equal(df, f)
        v2, f2, _ = api.extract_mesh(D, Wt, rig["origin"], rig["voxel"], mw)
        assert _bits_equal(v2, v) and np.array_equal(f2, f)
    print("%s, trunc %g voxels: %d valid voxels, %d vertices, %d faces, integrate %.2f ms" % (
        maps, trunc_vox, int((Wt > 0).sum()), len(v), len(f), info["integrate_ms"]))


@pytest.mark.parametrize("maps", ["gt", "pm"])
def test_gpu_mesh_does_not_depend_on_the_worlds_scale(rig, maps):
    """P's fourth column, the depths, the depth range, origin, voxel and trunc times 2^-10: the same D and Wt bits, the
    same faces, every vertex times 2^-10 exactly."""
    from gipuma_b200 import api
    s = 2.0 ** -10
    sPs = [np.hstack([np.asarray(P, np.float64)[:, :3], np.asarray(P, np.float64)[:, 3:] * s]) for P in rig["fPs"]]
    dep = rig["maps"][maps]
    trunc = 3.0 * rig["voxel"]
    D, Wt, _ = api.tsdf_integrate(dep, rig["fPs"], rig["origin"], rig["voxel"], rig["dims"], trunc, DMIN, DMAX,
                                  cam_scale=rig["scale"])
    so = tuple(x * s for x in rig["origin"])
    sD, sW, _ = api.tsdf_integrate(dep * np.float32(s), sPs, so, rig["voxel"] * s, rig["dims"], trunc * s, DMIN * s, DMAX * s,
                                   cam_scale=rig["scale"])
    assert _bits_equal(sD, D) and _bits_equal(sW, Wt)
    v, f, _ = api.extract_mesh(D, Wt, rig["origin"], rig["voxel"], 2)
    sv, sf, _ = api.extract_mesh(sD, sW, so, rig["voxel"] * s, 2)
    assert len(f) > 100 and np.array_equal(sf, f) and _bits_equal(sv, v * np.float32(s))


def _adversarial():
    rng = np.random.default_rng(11)
    out = []
    D = rng.standard_normal((5, 6, 7)).astype(np.float32)
    out.append(("all invalid", D, np.zeros(D.shape, np.uint16), 1))
    W = np.zeros((2, 2, 2), np.uint16)
    for m in (0, 1, 3, 7):                                     # the corners 0, x, x+y, 1 of tetrahedron xyz
        W[m >> 2 & 1, m >> 1 & 1, m & 1] = 1
    out.append(("one valid tetrahedron", np.array([[[-1, 2], [3, 4]], [[5, 6], [7, 0.5]]], np.float32), W, 1))
    for shape in ((2, 2, 2), (2, 3, 2), (3, 2, 5), (7, 9, 11), (2, 17, 3)):
        D = rng.standard_normal(shape).astype(np.float32)
        out.append(("dims %s" % (shape,), D, rng.integers(0, 4, shape).astype(np.uint16), 2))
    D = rng.standard_normal((9, 8, 7)).astype(np.float32)
    Wt = rng.integers(0, 3, D.shape).astype(np.uint16)
    D[Wt == 0] = np.float32("nan")
    out.append(("NaN where Wt = 0", D, Wt, 1))
    D = rng.choice(np.array([-0.0, 0.0, -1.0, 1.0, 1e-30, -1e-45], np.float32), (6, 7, 8))
    out.append(("zeros, signed zeros and denormals", D, np.ones(D.shape, np.uint16), 1))
    # long thin boxes, (nx, ny, nz) = (2048, 2, 3), (3, 2048, 2), (2, 3, 2048), and a 2048 x 2048 x 2 sheet: per-axis
    # neighbour offsets and many blocks per scan
    for shape in ((3, 2, 2048), (2, 2048, 3), (2048, 3, 2), (2, 2048, 2048)):
        D = rng.standard_normal(shape).astype(np.float32)
        out.append(("dims %s" % (shape[::-1],), D, rng.integers(0, 3, shape).astype(np.uint16), 1))
    # infinite, NaN and +-FLT_MAX values at valid points: dp - dq overflows, t is NaN or 0
    big = np.finfo(np.float32).max
    D = rng.choice(np.array([np.inf, -np.inf, np.nan, big, -big, 1.0, -1.0, -0.0], np.float32), (7, 8, 9))
    out.append(("inf, NaN and FLT_MAX at valid points", D, np.ones(D.shape, np.uint16), 1))
    # the largest weight: min_weight 65535 keeps the points at 65535, 65536 keeps none
    D = rng.standard_normal((6, 7, 8)).astype(np.float32)
    Wt = rng.choice(np.array([65535, 65534, 1], np.uint16), D.shape)
    out.append(("Wt 65535, min_weight 65535", D, Wt, 65535))
    out.append(("Wt 65535, min_weight 65536", D, Wt, 65536))
    return out


@pytest.mark.parametrize("case", range(len(_adversarial())))
def test_gpu_mesh_on_adversarial_volumes(case):
    import torch
    from gipuma_b200 import api
    from oracle import pymesh
    name, D, Wt, mw = _adversarial()[case]
    origin, voxel = (0.25, -3.0, 1.5), 0.75
    v, f, _ = api.extract_mesh(D, Wt, origin, voxel, mw)
    ov, of = pymesh.extract(D, Wt, origin, voxel, mw)
    # bit for bit, NaN equal to NaN: where dp - dq is inf - inf or overflows, the GPU's NaN is 0x7fffffff and the host's
    # keeps the sign and payload of the NaN it came from
    assert v.shape == ov.shape and bits_equal(v, ov) == 0 and np.array_equal(f, of), name
    dv, df, _ = api.extract_mesh(torch.from_numpy(D).cuda(), torch.from_numpy(Wt.astype(np.int32)).to(torch.uint16).cuda(),
                                 origin, voxel, mw)
    assert _bits_equal(dv, v) and np.array_equal(df, f), name
    if name == "all invalid":
        assert len(v) == 0 and len(f) == 0
    if name == "one valid tetrahedron":
        assert len(v) == 3 and len(f) == 1
    if name.startswith("Wt 65535"):
        assert (len(f) > 0) == (mw == 65535)


def test_gpu_tsdf_with_a_box_partly_behind_a_camera(rig):
    """A box reaching from behind the first camera to beyond the surface: voxels behind a camera (z <= 0) and outside its
    image take nothing from it; the GPU equals the restatement."""
    from gipuma_b200 import api
    from oracle import pymesh
    from gipuma_b200 import scene as S
    _, _, C0 = S.decompose_projection(rig["fPs"][0])
    o = rig["origin"]
    voxel = float(np.float32(rig["voxel"] * 4))
    origin = (o[0], o[1], float(np.float32(C0[2] - 20 * voxel)))
    dims = (24, 22, 40)
    P0 = np.asarray(rig["fPs"][0], np.float64)
    z = [origin[a] + (np.arange(dims[a]) + 0.5) * voxel for a in range(3)]
    Z, Y, X = np.meshgrid(z[2], z[1], z[0], indexing="ij")
    depth0 = P0[2, 0] * X + P0[2, 1] * Y + P0[2, 2] * Z + P0[2, 3]
    assert (depth0 <= 0).any() and (depth0 > 0).any()
    dep = rig["maps"]["gt"]
    D, Wt, _ = api.tsdf_integrate(dep, rig["fPs"], origin, voxel, dims, 3 * voxel, DMIN, DMAX, cam_scale=rig["scale"])
    oD, oW = _oracle_tsdf(dep, rig["fPs"], rig["scale"], origin, voxel, dims, 3 * voxel)
    assert _bits_equal(D, oD) and _bits_equal(Wt, oW)
    v, f, _ = api.extract_mesh(D, Wt, origin, voxel, 1)
    ov, of = pymesh.extract(D, Wt, origin, voxel, 1)
    assert _bits_equal(v, ov) and np.array_equal(f, of)


def test_gpu_mesh_capacity_and_counts():
    """A too-small capacity is refused after the whole run with both counts set; the retry with the counts fills."""
    import ctypes as C
    from gipuma_b200 import api
    rng = np.random.default_rng(3)
    D = rng.standard_normal((6, 7, 8)).astype(np.float32)
    Wt = np.ones(D.shape, np.uint16)
    lib = api.load_library()
    d = api.GpmMeshDesc(D.ctypes.data, Wt.ctypes.data, 0, (C.c_float * 3)(0, 0, 0), 1.0, (C.c_int * 3)(8, 7, 6), 1, 0)
    r = api.GpmMeshResult(0, 0, 0, 0, None, None, 0.0, 0.0)
    assert lib.gpm_mesh_extract(C.byref(d), C.byref(r)) == -1 and "capacity" in lib.gpm_last_error().decode()
    nv, nf = r.n_vertices, r.n_faces
    assert nv > 0 and nf > 0
    v = np.zeros((nv, 3), np.float32)
    f = np.zeros((nf - 1, 3), np.int32)
    r = api.GpmMeshResult(0, 0, nv, nf - 1, v.ctypes.data, f.ctypes.data, 0.0, 0.0)
    assert lib.gpm_mesh_extract(C.byref(d), C.byref(r)) == -1 and (r.n_vertices, r.n_faces) == (nv, nf)
    v2, f2, _ = api.extract_mesh(D, Wt, (0, 0, 0), 1.0, 1)
    assert _bits_equal(v, v2) and np.array_equal(f, f2[:nf - 1])


@pytest.fixture(scope="module")
def dtu():
    from gipuma_b200 import api, scene as S
    Ps = [S.load_dtu_projections()[i] for i in range(49)]
    H, W = 1200, 1600
    hf = S.HeightField(z0=550.0, unit=550.0 / S.prepare_cameras(Ps[:1])[0].fx, seed=77)
    gt = S.render_norm4(Ps, 1.0, H, W, hf)
    dep = np.ascontiguousarray(gt[..., 3])
    origin, voxel = _box(Ps, 1.0, H, W, hf, 512)
    return dict(Ps=Ps, hf=hf, dep=dep, origin=origin, voxel=voxel, gt=S.gt_points(Ps, 1.0, H, W, hf, stride=3, norm4=gt))


def test_gpu_mesh_at_dtu_size(dtu):
    """49 ground-truth maps at 1600 x 1200 into a 512^3 box: slabs of the volume equal the restatement, and so do meshes
    of slabs of it; the mesh of the whole box lies within a voxel of the ground truth at the 95th percentile."""
    import torch
    from gipuma_b200 import api
    from oracle import pymesh
    dims = (512, 512, 512)
    trunc = 3.0 * dtu["voxel"]
    dd = torch.from_numpy(dtu["dep"]).cuda()
    D, Wt, info = api.tsdf_integrate(dd, dtu["Ps"], dtu["origin"], dtu["voxel"], dims, trunc, DMIN, DMAX)
    Dh, Wh = D.cpu().numpy(), Wt.cpu().numpy()
    filled = np.nonzero((Wh > 0).any(axis=(1, 2)))[0]
    assert len(filled) > 20
    rng = np.random.default_rng(2026)
    for k0 in sorted(rng.choice(filled[:-4], 3, replace=False)):
        k0 = int(k0)
        oD, oW = _oracle_tsdf(dtu["dep"], dtu["Ps"], 1.0, dtu["origin"], dtu["voxel"], dims, trunc, (k0, k0 + 4))
        assert _bits_equal(Dh[k0:k0 + 4], oD) and _bits_equal(Wh[k0:k0 + 4], oW), k0
        so = (dtu["origin"][0], dtu["origin"][1], float(np.float32(dtu["origin"][2] + k0 * dtu["voxel"])))
        v, f, _ = api.extract_mesh(np.ascontiguousarray(Dh[k0:k0 + 4]), np.ascontiguousarray(Wh[k0:k0 + 4]), so, dtu["voxel"], 2)
        ov, of = pymesh.extract(Dh[k0:k0 + 4], Wh[k0:k0 + 4], so, dtu["voxel"], 2)
        assert _bits_equal(v, ov) and np.array_equal(f, of), k0
    v, f, minfo = api.extract_mesh(D, Wt, dtu["origin"], dtu["voxel"], 2)
    v2, f2, _ = api.extract_mesh(D, Wt, dtu["origin"], dtu["voxel"], 2)
    assert _bits_equal(v, v2) and np.array_equal(f, f2)
    pts = api.sample_mesh(v, f, dtu["voxel"] / 2)
    d, _ = api.nearest_distance(pts, dtu["gt"], 20.0 * dtu["voxel"])
    p95 = float(np.percentile(d, 95))
    print("DTU size: voxel %.4f, integrate %.1f ms, extract %.1f ms, %d vertices, %d faces, %d samples, accuracy p50 %.4f "
          "p95 %.4f voxels" % (dtu["voxel"], info["integrate_ms"], minfo["extract_ms"], len(v), len(f), len(pts),
                               np.percentile(d, 50) / dtu["voxel"], p95 / dtu["voxel"]))
    assert p95 <= dtu["voxel"]

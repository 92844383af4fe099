"""The meshing (DESIGN.md §24) without a GPU: the C restatement (oracle/mesh_oracle.c) on volumes with known answers — a
plane half-way between lattice layers, a closed consistently oriented sphere, an invalid corner, -0.0 and exact zeros — the
Kuhn split's agreement on shared cube faces, the integration's rules on a hand-made rig, the PLY mesh layout byte for byte,
the struct layouts, and every refusal of the C-ABI and of the Python API."""
import ctypes as C
import os
import subprocess
from collections import Counter

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PERMS = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]        # DESIGN.md §24: xyz, xzy, yxz, yzx, zxy, zyx


def _extract(D, Wt, origin=(0.0, 0.0, 0.0), voxel=1.0, min_weight=1):
    from oracle import pymesh
    return pymesh.extract(np.asarray(D, np.float32), np.asarray(Wt, np.uint16), origin, voxel, min_weight)


def _centres(n, origin, voxel):
    """Lattice coordinates per axis as the kernels compute them: origin + (i + 0.5) * voxel in float32."""
    return [np.float32(origin[a]) + (np.arange(n[a], dtype=np.float32) + np.float32(0.5)) * np.float32(voxel) for a in range(3)]


def _sphere(n=(13, 14, 15), c=(6.3, 6.9, 7.2), r=4.6, origin=(0.0, 0.0, 0.0), voxel=1.0):
    x, y, z = _centres(n, origin, voxel)
    Z, Y, X = np.meshgrid(z.astype(np.float64), y.astype(np.float64), x.astype(np.float64), indexing="ij")
    D = (np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r).astype(np.float32)
    return D, np.ones(D.shape, np.uint16)


def _directed_edges(f):
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def _signed_volume(v, f):
    a, b, c = (v[f[:, k]].astype(np.float64) for k in range(3))
    return np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0


def test_a_plane_half_way_between_layers_puts_every_vertex_on_it():
    """D = z - 2 on the lattice z = 0.5, 1.5, 2.5, ...: every crossing edge has t = 1/2 exactly, so every vertex has z = 2,
    and the faces point to +z, the outside."""
    n = (7, 6, 5)
    x, y, z = _centres(n, (0, 0, 0), 1.0)
    D = np.broadcast_to((z - np.float32(2.0))[:, None, None], (n[2], n[1], n[0])).astype(np.float32)
    v, f = _extract(D, np.ones(D.shape, np.uint16))
    assert len(v) > 0 and len(f) > 0
    assert (v[:, 2] == np.float32(2.0)).all()
    nrm = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert (nrm[:, 2] > 0).all() and (np.abs(nrm[:, :2]) == 0).all()
    # the plane covers the (nx - 1) x (ny - 1) cells of the box: two triangles' worth of area per cell
    assert np.isclose(0.5 * nrm[:, 2].sum(), (n[0] - 1) * (n[1] - 1))


@pytest.mark.parametrize("voxel", [1.0, 0.37])
def test_a_sphere_is_a_closed_consistently_oriented_two_manifold(voxel):
    o = (-1.25, 0.5, 2.0)
    c = tuple(o[a] + 7.0 * voxel + 0.3 * a * voxel for a in range(3))
    D, Wt = _sphere(origin=o, voxel=voxel, c=c, r=4.6 * voxel)
    v, f = _extract(D, Wt, o, voxel)
    # every directed edge once, its reverse once: each undirected edge in exactly two faces, traversed in opposite directions
    de = _directed_edges(f)
    assert len(set(map(tuple, de))) == len(de)
    assert set(map(tuple, de)) == set(map(tuple, de[:, ::-1]))
    E = len(de) // 2
    assert len(v) - E + len(f) == 2
    # every vertex is used, no face repeats a vertex
    assert set(np.unique(f)) == set(range(len(v)))
    assert (f[:, 0] != f[:, 1]).all() and (f[:, 1] != f[:, 2]).all() and (f[:, 0] != f[:, 2]).all()
    # outward: counter-clockwise seen from outside gives a positive enclosed volume near the sphere's
    vol = _signed_volume(v, f)
    assert 0.9 < vol / (4.0 / 3.0 * np.pi * (4.6 * voxel) ** 3) < 1.0
    dist = np.abs(np.linalg.norm(v.astype(np.float64) - np.array(c), axis=1) - 4.6 * voxel)
    assert dist.max() < voxel


def test_faces_point_to_the_outside_at_every_face():
    """Each face's normal has a positive component along the outward radial direction of the sphere."""
    D, Wt = _sphere()
    v, f = _extract(D, Wt)
    ctr = v[f].mean(axis=1).astype(np.float64) - np.array((6.3, 6.9, 7.2))
    nrm = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]).astype(np.float64)
    big = np.linalg.norm(nrm, axis=1) > 1e-3
    assert (np.einsum("ij,ij->i", nrm, ctr)[big] > 0).all()


def _edge_vertex(D, p, q, origin, voxel):
    """The vertex of edge p -> q ((i, j, k) lattice points, p lower) as DESIGN.md §24 computes it, in numpy float32."""
    dp, dq = D[p[2], p[1], p[0]], D[q[2], q[1], q[0]]
    t = np.float32(dp / np.float32(dp - dq))
    out = []
    for a in range(3):
        xp = np.float32(origin[a]) + (np.float32(p[a]) + np.float32(0.5)) * np.float32(voxel)
        xq = np.float32(origin[a]) + (np.float32(q[a]) + np.float32(0.5)) * np.float32(voxel)
        out.append(np.float32(xp + np.float32(t * np.float32(xq - xp))))
    return tuple(out)


def test_an_invalid_corner_removes_exactly_its_tetrahedra():
    """A point made invalid removes every face with a vertex on one of its edges (the faces of the tetrahedra that have it
    as a corner) and nothing else; the other faces keep their order."""
    D, Wt = _sphere()
    v0, f0 = _extract(D, Wt)
    p = (int(round(6.3 + 4.6 - 0.5)), 6, 6)                        # a point next to the surface, on the +x side
    assert D[p[2], p[1], p[0]] * D[p[2], p[1], p[0] + 1] < 0
    near = set()
    for m in range(1, 8):
        e = np.array([m & 1, m >> 1 & 1, m >> 2 & 1])
        for lo, hi in ((np.array(p), np.array(p) + e), (np.array(p) - e, np.array(p))):
            near.add(_edge_vertex(D, tuple(lo), tuple(hi), (0, 0, 0), 1.0))
    Wt1 = Wt.copy()
    Wt1[p[2], p[1], p[0]] = 0
    v1, f1 = _extract(D, Wt1)
    key = lambda v, f: [tuple(tuple(x) for x in v[t].tolist()) for t in f]
    k0 = key(v0, f0)
    kept = [t for t in k0 if not any(tuple(np.float32(c) for c in x) in near for x in t)]
    assert len(kept) < len(k0)
    assert key(v1, f1) == kept


def test_zero_and_negative_zero_are_outside():
    """A point is inside when D < 0: -0.0 and +0.0 are outside, alike.  One inside corner of a cube whose other corners
    are 0 gives its 6 tetrahedra's 6 triangles on the 7 edges from it, each vertex on the far corner (t = 1)."""
    for z in (0.0, -0.0):
        D = np.full((2, 2, 2), z, np.float32)
        v, f = _extract(D, np.ones((2, 2, 2), np.uint16))
        assert len(v) == 0 and len(f) == 0
        D[0, 0, 0] = -1.0
        v, f = _extract(D, np.ones((2, 2, 2), np.uint16))
        assert len(v) == 7 and len(f) == 6
        assert {tuple(x) for x in v.tolist()} == {(0.5 + i, 0.5 + j, 0.5 + k) for i in (0, 1) for j in (0, 1) for k in (0, 1)} - {(0.5, 0.5, 0.5)}
    # all inside but one corner at -0.0: that corner is outside
    D = np.full((2, 2, 2), -1.0, np.float32)
    D[1, 1, 1] = -0.0
    v, f = _extract(D, np.ones((2, 2, 2), np.uint16))
    assert len(v) == 7 and len(f) == 6
    assert (v == np.float32(1.5)).all()                            # t = -1 / (-1 - -0) = 1: every vertex on the far corner
    assert _signed_volume(v, f) == 0.0                             # degenerate, yet...
    de = _directed_edges(f)
    assert len(set(map(tuple, de))) == len(de)                     # ...consistently wound


def test_the_kuhn_split_agrees_on_shared_cube_faces():
    """The tetrahedra of DESIGN.md §24 tile the cube (each of volume 1/6, signed by its permutation's parity), and the
    triangles they put on a cube face are those the neighbouring cube puts on it."""
    def tets():
        for a, b, c in PERMS:
            yield [0, 1 << a, (1 << a) | (1 << b), 7]

    pos = lambda m: np.array([m & 1, m >> 1 & 1, m >> 2 & 1])
    for t, (a, b, c) in zip(tets(), PERMS):
        vol = np.linalg.det(np.stack([pos(t[1]), pos(t[2]), pos(t[3])]).astype(float))
        sign = np.linalg.det(np.eye(3)[[a, b, c]])
        assert np.isclose(vol, sign)
    for axis in range(3):
        for side in (0, 1):
            # triangles of tetrahedron faces lying on the plane axis = side of the cube at the origin
            tri = set()
            for t in tets():
                for skip in range(4):
                    f = [m for k, m in enumerate(t) if k != skip]
                    if all(pos(m)[axis] == side for m in f):
                        tri.add(frozenset(tuple(pos(m)) for m in f))
            assert len(tri) == 2
            if side == 0:
                low = tri
            else:
                e = pos(1 << axis)
                assert {frozenset(tuple(np.array(x) - e) for x in s) for s in tri} == low


def test_random_volumes_are_watertight_inside_the_box():
    """A random field, every point valid: every edge of the mesh off the box's boundary is in exactly two faces, in
    opposite directions."""
    rng = np.random.default_rng(5)
    D = rng.standard_normal((9, 10, 11)).astype(np.float32)
    v, f = _extract(D, np.ones(D.shape, np.uint16))
    de = _directed_edges(f)
    c = Counter(map(tuple, de))
    assert max(c.values()) == 1
    lo, hi = np.float32(0.5), np.float32(np.array([11, 10, 9], np.float32) - 0.5)
    for a, b in de:
        if (a, b) in c and (b, a) not in c:
            pa, pb = v[a], v[b]
            on_boundary = any((pa[k] == lo and pb[k] == lo) or (pa[k] == hi[k] and pb[k] == hi[k]) for k in range(3))
            assert on_boundary


def test_min_weight_and_the_number_of_valid_corners():
    from oracle import pymesh
    D, Wt = _sphere()
    Wt = np.where(np.arange(D.size).reshape(D.shape) % 7 == 0, 1, 3).astype(np.uint16)
    v1, f1 = pymesh.extract(D, Wt, (0, 0, 0), 1.0, 1)
    v3, f3 = pymesh.extract(D, Wt, (0, 0, 0), 1.0, 3)
    v4, f4 = pymesh.extract(D, Wt, (0, 0, 0), 1.0, 4)
    assert len(f3) < len(f1) and len(v4) == 0 and len(f4) == 0


def _P(c=(0.0, 0.0, 0.0), F=50.0, W=20, H=16):
    K = np.array([[F, 0, W / 2], [0, F, H / 2], [0, 0, 1.0]])
    return K @ np.hstack([np.eye(3), -np.array(c, dtype=np.float64)[:, None]])


def test_integration_rules_on_a_hand_made_rig():
    """Two cameras on the z axis looking at the plane z = 10: S / Wt is the truncated, normalised signed distance along z,
    invalid and out-of-range depths are skipped, a voxel behind the surface by more than trunc gets nothing from a view."""
    from gipuma_b200 import api
    from oracle import pymesh
    W, H = 20, 16
    Ps = [_P(), _P((0.0, 0.0, 2.0))]
    dep = np.stack([np.full((H, W), 10.0, np.float32), np.full((H, W), 8.0, np.float32)])
    dep[1, :, :4] = 0.0                                        # invalid
    dep[1, :, 4:6] = 500.0                                     # outside the depth range
    cams = api.fuse_cameras(Ps)
    origin, voxel, dims = (-0.5, -0.5, 6.0), 0.5, (2, 2, 16)
    D, Wt = pymesh.tsdf(dep, cams, origin, voxel, dims, 1.5, 1.0, 100.0)
    z = np.float32(6.0) + (np.arange(16, dtype=np.float32) + np.float32(0.5)) * np.float32(0.5)
    want = np.clip((np.float32(10.0) - z) / np.float32(1.5), None, 1.0).astype(np.float32)
    ok = z - np.float32(10.0) <= np.float32(1.5)
    col = D[:, 0, 0]
    assert np.array_equal(Wt[:, 0, 0], np.where(ok, 2, 0))
    assert np.allclose(col[ok], want[ok], atol=1e-6) and np.isnan(col[~ok]).all()
    assert D[~ok, 0, 0].view(np.uint32).tolist() == [0x7FFFFFFF] * int((~ok).sum())
    # the voxels that fall on view 1's invalid or out-of-range pixels take view 0 only
    D2, Wt2 = pymesh.tsdf(dep, cams, (-1.05, -0.5, 9.0), 0.1, (2, 2, 2), 1.5, 1.0, 100.0)
    assert (Wt2 == 1).all()


def test_ply_mesh_header_byte_for_byte(tmp_path):
    from gipuma_b200 import api
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)
    p = str(tmp_path / "m.ply")
    api.write_ply_mesh(p, v, f)
    data = open(p, "rb").read()
    header = (b"ply\nformat binary_little_endian 1.0\nelement vertex 4\nproperty float x\nproperty float y\n"
              b"property float z\nelement face 4\nproperty list uchar int vertex_indices\nend_header\n")
    assert data[:len(header)] == header
    body = v.astype("<f4").tobytes() + b"".join(b"\x03" + t.astype("<i4").tobytes() for t in f)
    assert data[len(header):] == body
    rv, rf = api.read_ply_mesh(p)
    assert rv.tobytes() == v.tobytes() and np.array_equal(rf, f)
    api.write_ply_mesh(str(tmp_path / "e.ply"), np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    assert open(tmp_path / "e.ply", "rb").read() == header.replace(b"vertex 4", b"vertex 0").replace(b"face 4", b"face 0")
    with pytest.raises(ValueError, match="face index"):
        api.write_ply_mesh(p, v, f + 1)
    lib = api.load_library()
    bad = np.array([[0, 1, 4]], np.int32)
    assert lib.gpm_write_ply_mesh(p.encode(), v.ctypes.data, 4, bad.ctypes.data, 1) == -1
    assert lib.gpm_write_ply_mesh(p.encode(), None, 4, f.ctypes.data, 4) == -1
    assert lib.gpm_write_ply_mesh(p.encode(), v.ctypes.data, -1, None, 0) == -1


def test_sample_mesh_is_a_barycentric_lattice():
    from gipuma_b200 import api
    v = np.array([[0, 0, 0], [3, 0, 0], [0, 2, 0], [0, 0, 0.5]], np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]], np.int32)
    s = api.sample_mesh(v, f, 1.0)
    # face 0: longest edge sqrt(13) -> n = 4, 15 points; face 1: sqrt(4.25) -> n = 3, 10 points
    assert s.shape == (25, 3) and s.dtype == np.float32
    assert np.array_equal(s[0], v[0]) and np.array_equal(s[4], v[2]) and np.array_equal(s[14], v[1])
    assert np.array_equal(api.sample_mesh(v, f, 1.0), s)
    assert (s[:15, 0] / 3 + s[:15, 1] / 2 <= 1 + 1e-6).all()
    with pytest.raises(ValueError):
        api.sample_mesh(v, f, 0.0)


def test_mesh_layouts_match_ctypes(tmp_path):
    from gipuma_b200 import api
    fields = {"gpm_tsdf_desc": (api.GpmTsdfDesc, ["n_views", "width", "height", "depth", "on_device", "P", "cam_scale",
                                                  "depth_min", "depth_max", "origin", "voxel", "dims", "trunc", "device"]),
              "gpm_tsdf_result": (api.GpmTsdfResult, ["D", "weight", "upload_ms", "integrate_ms"]),
              "gpm_mesh_desc": (api.GpmMeshDesc, ["D", "weight", "on_device", "origin", "voxel", "dims", "min_weight", "device"]),
              "gpm_mesh_result": (api.GpmMeshResult, ["n_vertices", "n_faces", "vertex_capacity", "face_capacity", "vertices",
                                                      "faces", "upload_ms", "extract_ms"])}
    prints, want = [], []
    for s, (cls, names) in fields.items():
        prints.append('printf("%%zu\\n", sizeof(%s));' % s)
        want.append(C.sizeof(cls))
        for nm in names:
            prints.append('printf("%%zu\\n", offsetof(%s, %s));' % (s, nm))
            want.append(getattr(cls, nm).offset)
    prints.append('printf("%d\\n", GPM_MESH_MAX_DIM);')
    want.append(api.MESH_MAX_DIM)
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gipuma_b200.h"\nint main(void){ %s return 0; }\n'
                   % " ".join(prints))
    exe = str(tmp_path / "t")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    assert [int(x) for x in subprocess.check_output([exe]).split()] == want


def _tsdf_desc(api, dep, Pm, **kw):
    d = api.GpmTsdfDesc(2, 20, 16, dep.ctypes.data, 0, Pm.ctypes.data_as(C.POINTER(C.c_double)), 1.0, 1.0, 100.0,
                        (C.c_float * 3)(0, 0, 0), 0.5, (C.c_int * 3)(4, 4, 4), 1.5, 0)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_bad_arguments_are_refused_before_any_cuda_call():
    from conftest import have_cuda
    from gipuma_b200 import api
    lib = api.load_library()
    nan, inf = float("nan"), float("inf")
    dep = np.full((2, 16, 20), 10.0, np.float32)
    P = np.ascontiguousarray(np.stack([_P(), _P((0, 0, 2.0))]).reshape(-1))
    out = np.zeros(64, np.float32)
    w = np.zeros(64, np.uint16)
    f3, i3 = C.c_float * 3, C.c_int * 3
    tsdf_bad = [(dict(n_views=0), "n_views"), (dict(n_views=257), "n_views"), (dict(width=0), "bad image size"),
                (dict(height=1 << 16, width=1 << 15), "bad image size"), (dict(depth=None), "required"),
                (dict(P=None), "required"), (dict(dims=i3(1, 4, 4)), "dims"), (dict(dims=i3(4, 2049, 4)), "dims"),
                (dict(dims=i3(2048, 2048, 1024)), "2^31 - 1"), (dict(origin=f3(0, nan, 0)), "origin"),
                (dict(origin=f3(inf, 0, 0)), "origin"), (dict(cam_scale=0.0), "bad projection matrix")]
    tsdf_bad += [(dict(voxel=x), "voxel") for x in (0.0, -1.0, nan, inf)]
    tsdf_bad += [(dict(trunc=x), "trunc") for x in (0.0, -1.0, nan, inf)]
    tsdf_bad += [(dict(depth_min=a, depth_max=b), "depth_min") for a, b in ((-1.0, 5.0), (5.0, 5.0), (6.0, 5.0), (nan, 5.0),
                                                                            (1.0, inf), (1.0, nan))]
    for kw, msg in tsdf_bad:
        r = api.GpmTsdfResult(out.ctypes.data, w.ctypes.data, 0.0, 0.0)
        rc = lib.gpm_tsdf_integrate(C.byref(_tsdf_desc(api, dep, P, **kw)), C.byref(r))
        got = lib.gpm_last_error().decode()
        assert rc == -1 and got.startswith("gpm_tsdf_integrate: ") and msg in got, (kw, rc, got)
    for res in (api.GpmTsdfResult(None, w.ctypes.data, 0.0, 0.0), api.GpmTsdfResult(out.ctypes.data, None, 0.0, 0.0)):
        assert lib.gpm_tsdf_integrate(C.byref(_tsdf_desc(api, dep, P)), C.byref(res)) == -1
    assert lib.gpm_tsdf_integrate(None, None) == -1

    D = np.zeros(64, np.float32)
    vb, fb = np.zeros(30, np.float32), np.zeros(30, np.int32)

    def mesh_call(res=None, **kw):
        d = api.GpmMeshDesc(D.ctypes.data, w.ctypes.data, 0, f3(0, 0, 0), 1.0, i3(4, 4, 4), 1, 0)
        for k, v in kw.items():
            setattr(d, k, v)
        r = res or api.GpmMeshResult(0, 0, 10, 10, vb.ctypes.data, fb.ctypes.data, 0.0, 0.0)
        return lib.gpm_mesh_extract(C.byref(d), C.byref(r)), lib.gpm_last_error().decode()

    mesh_bad = [(dict(D=None), "required"), (dict(weight=None), "required"), (dict(dims=i3(4, 4, 1)), "dims"),
                (dict(dims=i3(4, 4, 2049)), "dims"), (dict(dims=i3(2048, 2048, 2048)), "2^31 - 1"),
                (dict(origin=f3(0, 0, nan)), "origin"), (dict(min_weight=0), "min_weight"), (dict(min_weight=-3), "min_weight")]
    mesh_bad += [(dict(voxel=x), "voxel") for x in (0.0, -1.0, nan, inf)]
    for kw, msg in mesh_bad:
        rc, got = mesh_call(**kw)
        assert rc == -1 and got.startswith("gpm_mesh_extract: ") and msg in got, (kw, rc, got)
    for res in (api.GpmMeshResult(0, 0, -1, 10, vb.ctypes.data, fb.ctypes.data, 0.0, 0.0),
                api.GpmMeshResult(0, 0, 10, -1, vb.ctypes.data, fb.ctypes.data, 0.0, 0.0),
                api.GpmMeshResult(0, 0, 10, 10, None, fb.ctypes.data, 0.0, 0.0),
                api.GpmMeshResult(0, 0, 10, 10, vb.ctypes.data, None, 0.0, 0.0)):
        rc, got = mesh_call(res)
        assert rc == -1 and "bad result buffers" in got
    if not have_cuda():
        # valid descriptors reach the device, which is not there
        r = api.GpmTsdfResult(out.ctypes.data, w.ctypes.data, 0.0, 0.0)
        assert lib.gpm_tsdf_integrate(C.byref(_tsdf_desc(api, dep, P)), C.byref(r)) == -2
        assert mesh_call()[0] == -2
        assert mesh_call(api.GpmMeshResult(0, 0, 0, 0, None, None, 0.0, 0.0))[0] == -2


def test_api_refuses_bad_arguments_before_the_library_loads(monkeypatch):
    from gipuma_b200 import api

    def boom():
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(api, "load_library", boom)
    nan, inf = float("nan"), float("inf")
    dep = np.full((2, 16, 20), 10.0, np.float32)
    Ps = [_P(), _P((0, 0, 2.0))]
    good = dict(origin=(0, 0, 0), voxel=0.5, dims=(4, 4, 4), trunc=1.5, depth_min=1.0, depth_max=100.0)
    cases = [(dict(origin=(0, 0)), "origin"), (dict(origin=(0, nan, 0)), "origin"), (dict(origin=(1e39, 0, 0)), "origin"),
             (dict(dims=(4, 4)), "dims"), (dict(dims=(1, 4, 4)), "dims"), (dict(dims=(4, 4, 2049)), "dims"),
             (dict(dims=(2048, 2048, 1024)), "2\\^31 - 1"), (dict(voxel=0.0), "voxel"), (dict(voxel=nan), "voxel"),
             (dict(voxel=1e-50), "voxel"), (dict(trunc=-1.0), "trunc"), (dict(trunc=inf), "trunc"),
             (dict(depth_min=-1.0), "depth_min"), (dict(depth_min=200.0), "depth_min"), (dict(depth_max=inf), "depth_min")]
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            api.tsdf_integrate(dep, Ps, **dict(good, **kw))
    with pytest.raises(ValueError, match="cam_scale"):
        api.tsdf_integrate(dep, Ps, cam_scale=0.0, **good)
    for d, P in ((dep[0], Ps[:1]), (dep, Ps[:1]), (np.zeros((257, 2, 2), np.float32), Ps * 128 + Ps[:1])):
        with pytest.raises(ValueError, match="depth must be"):
            api.tsdf_integrate(d, P, **good)
    D, Wt = np.zeros((4, 4, 4), np.float32), np.zeros((4, 4, 4), np.uint16)
    ex = [((D, Wt, (0, 0, 0), 1.0, 0), ValueError, "min_weight"), ((D, Wt, (0, 0, 0), 1.0, 1.5), ValueError, "min_weight"),
          ((D, Wt[:3], (0, 0, 0), 1.0, 1), ValueError, "one shape"), ((D[0], Wt[0], (0, 0, 0), 1.0, 1), ValueError, "one shape"),
          ((D, Wt, (0, 0, 0), -1.0, 1), ValueError, "voxel"), ((D, Wt, (0, nan, 0), 1.0, 1), ValueError, "origin"),
          ((D[:1], Wt[:1], (0, 0, 0), 1.0, 1), ValueError, "dims"),
          ((D.astype(np.float64), Wt, (0, 0, 0), 1.0, 1), TypeError, "float32"),
          ((D, Wt.astype(np.int32), (0, 0, 0), 1.0, 1), TypeError, "uint16")]
    for args, err, msg in ex:
        with pytest.raises(err, match=msg):
            api.extract_mesh(*args)
    with pytest.raises(ValueError, match="min_weight"):
        api.mesh(dep, Ps, min_weight=0, **good)
    assert set(api.MESH_DEFAULTS) == {"trunc_voxels", "min_weight"}

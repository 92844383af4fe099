"""The planar prior's host code as it ships (gipuma_b200/csrc/gpm_prior.cpp, DESIGN.md §18), without a device.

gpm::delaunay and gpm::triangle_plane only run inside gpm_build_planar_prior, on support points in general position.  Here
an extern "C" shim around them is compiled with the unmodified gpm_prior.cpp under the library's host flags and loaded with
ctypes, and its output is compared element for element with oracle/pyprior.py on the inputs where a triangulation breaks:
collinear chains, lattices whose every quadrilateral is cocircular, points on hull edges and on a chain's extension, every
insertion order of a grid, random sets and lattices at the 4096-pixel coordinate bound.  The shipped triangulation must
also have empty circles and cover exactly the convex hull.  Its triangle planes must equal pyprior's bit for bit, also
where the cross product is zero, where the normal is flipped towards the camera and where a plane almost contains a ray."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pyprior  # noqa: E402

SHIM = r"""
#include <array>
#include <exception>
#include <vector>
namespace gpm {
std::vector<std::array<int, 3>> delaunay(const std::vector<int>& xy);
std::array<float, 4> triangle_plane(const float* Kinv, const int* x, const int* y, const float* const* plane);
}
// triangles into out[3 * cap]; returns their number, -1 when the triangulation throws, -2 when cap is too small
extern "C" long long shim_delaunay(const int* xy, long long n, int* out, long long cap)
{
    std::vector<std::array<int, 3>> t;
    try { t = gpm::delaunay(std::vector<int>(xy, xy + 2 * n)); } catch (const std::exception&) { return -1; }
    if ((long long)t.size() > cap) return -2;
    for (size_t i = 0; i < t.size(); i++)
        for (int k = 0; k < 3; k++) out[3 * i + k] = t[i][k];
    return (long long)t.size();
}
// planes: the three vertices' planes, 12 floats
extern "C" void shim_triangle_plane(const float* Kinv, const int* x, const int* y, const float* planes, float* out)
{
    const float* p[3] = {planes, planes + 4, planes + 8};
    const std::array<float, 4> q = gpm::triangle_plane(Kinv, x, y, p);
    for (int k = 0; k < 4; k++) out[k] = q[k];
}
"""


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    gxx = shutil.which("g++")
    assert gxx, "g++ is needed to build gpm_prior.cpp for the host"
    d = tmp_path_factory.mktemp("prior_shim")
    src = d / "shim.cpp"
    src.write_text(SHIM)
    out = d / "libprior_shim.so"
    # the host flags the library build passes for gpm_prior.cpp (gipuma_b200/build.py: -O3 -std=c++17 -fPIC -shared)
    subprocess.check_call([gxx, "-O3", "-std=c++17", "-fPIC", "-shared", "-o", str(out), str(src),
                           os.path.join(ROOT, "gipuma_b200", "csrc", "gpm_prior.cpp")])
    lib = C.CDLL(str(out))
    lib.shim_delaunay.restype = C.c_longlong
    lib.shim_delaunay.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong]
    lib.shim_triangle_plane.restype = None
    lib.shim_triangle_plane.argtypes = [C.c_void_p] * 5
    return lib


def cpp_delaunay(lib, pts):
    xy = np.ascontiguousarray(np.asarray(pts, np.int32).reshape(-1, 2))
    cap = max(2 * len(xy), 1)
    out = np.zeros((cap, 3), np.int32)
    n = lib.shim_delaunay(xy.ctypes.data, len(xy), out.ctypes.data, cap)
    assert n >= 0, "gpm::delaunay failed (%d)" % n
    return out[:n].astype(np.int64)


def cpp_triangle_plane(lib, Kinv, xs, ys, planes):
    k = np.ascontiguousarray(np.asarray(Kinv, np.float32).ravel())
    x = np.ascontiguousarray(np.asarray(xs, np.int32))
    y = np.ascontiguousarray(np.asarray(ys, np.int32))
    p = np.ascontiguousarray(np.asarray(planes, np.float32).reshape(12))
    out = np.zeros(4, np.float32)
    lib.shim_triangle_plane(k.ctypes.data, x.ctypes.data, y.ctypes.data, p.ctypes.data, out.ctypes.data)
    return out


# ---- triangulation ----------------------------------------------------------------------------------------------------
def incircle_many(P, tris, chunk=512):
    """max over the points of every triangle's exact in-circle determinant, excluding its own vertices (int64: coordinates
    <= 4096 keep the determinant below 2^53)"""
    worst = np.iinfo(np.int64).min
    for s in range(0, len(tris), chunk):
        t = tris[s:s + chunk]
        a, b, c = (P[t[:, i]][:, None, :] for i in range(3))
        d = P[None, :, :]
        adx, ady = a[..., 0] - d[..., 0], a[..., 1] - d[..., 1]
        bdx, bdy = b[..., 0] - d[..., 0], b[..., 1] - d[..., 1]
        cdx, cdy = c[..., 0] - d[..., 0], c[..., 1] - d[..., 1]
        det = ((adx * adx + ady * ady) * (bdx * cdy - cdx * bdy) + (bdx * bdx + bdy * bdy) * (cdx * ady - adx * cdy) +
               (cdx * cdx + cdy * cdy) * (adx * bdy - bdx * ady))
        own = np.arange(len(P))[None, :]
        det[(own == t[:, :1]) | (own == t[:, 1:2]) | (own == t[:, 2:3])] = np.iinfo(np.int64).min
        worst = max(worst, int(det.max()))
    return worst


def hull_area2(P):
    """twice the convex hull's area, exactly (0 for fewer than three points or collinear ones)"""
    if len(P) < 3:
        return 0
    u = P - P[0]
    if not (u[1, 0] * u[:, 1] - u[1, 1] * u[:, 0]).any():      # every point on the line through the first two
        return 0
    from scipy.spatial import ConvexHull
    hv = P[ConvexHull(P.astype(float)).vertices]                  # counter-clockwise
    return int(sum(hv[i, 0] * hv[(i + 1) % len(hv), 1] - hv[(i + 1) % len(hv), 0] * hv[i, 1] for i in range(len(hv))))


def check_same(lib, pts):
    """gpm::delaunay == pyprior.delaunay element for element; empty circles; twice the area == the hull's"""
    pts = [(int(x), int(y)) for x, y in pts]
    assert len(set(pts)) == len(pts)
    got = cpp_delaunay(lib, pts)
    want = pyprior.delaunay(pts)
    assert got.shape == want.shape and np.array_equal(got, want), (len(pts), got.shape, want.shape)
    P = np.asarray(pts, np.int64).reshape(-1, 2)
    if len(got):
        o = [(P[b, 0] - P[a, 0]) * (P[c, 1] - P[a, 1]) - (P[b, 1] - P[a, 1]) * (P[c, 0] - P[a, 0]) for a, b, c in got]
        o = np.asarray(o, np.int64)
        assert (o > 0).all()                                       # counter-clockwise, none degenerate
        assert incircle_many(P, got) <= 0                          # no point strictly inside any circumcircle
        assert int(o.sum()) == hull_area2(P)
    else:
        assert hull_area2(P) == 0
    return got


def degenerate_set(kind):
    """the sets of test_planar_prior.py's test_delaunay_degenerate_sets"""
    if kind == "rows":
        return [(x, y) for y in (0, 7, 14) for x in range(0, 60, 5)]
    if kind == "grid":
        return [(x, y) for y in range(0, 50, 5) for x in range(0, 50, 5)]
    if kind == "cocircular":
        return [(0, 0), (10, 0), (10, 10), (0, 10), (5, 5), (5, -5), (15, 5), (5, 15), (-5, 5), (8, 1), (2, 9)]
    if kind == "collinear_start":
        return [(x, 3) for x in range(0, 40, 3)] + [(17, 20), (4, 0), (33, 1), (20, -9)]
    rng = np.random.default_rng(7)
    pts = [(min(5 * cx + int(rng.integers(0, 2)) * 4, 61), 5 * cy + int(rng.integers(0, 5))) for cy in range(9) for cx in range(13)]
    return list(dict.fromkeys(pts))


@pytest.mark.parametrize("kind", ["rows", "grid", "cocircular", "collinear_start", "border"])
def test_degenerate_sets_equal_the_restatement(shim, kind):
    pts = degenerate_set(kind)
    if kind == "cocircular":                 # pyprior's own test has negative coordinates; the library's range is 0..4096
        pts = [(x + 5, y + 5) for x, y in pts]
    assert len(check_same(shim, pts)) > 0


@pytest.mark.parametrize("pts", [[], [(7, 9)], [(1, 1), (2, 2)], [(x, 2 * x) for x in range(10)],
                                 [(3 * x, 4096) for x in range(0, 1366, 7)], [(0, y) for y in range(4096, -1, -512)]],
                         ids=["empty", "one", "two", "diagonal", "bottom_row", "left_column_descending"])
def test_fewer_than_three_or_collinear_give_no_triangles(shim, pts):
    assert len(check_same(shim, pts)) == 0


@pytest.mark.parametrize("order", ["row_major", "reversed", "column_major", "shuffled_0", "shuffled_1", "shuffled_2"])
def test_grid_in_every_order(shim, order):
    pts = [(x, y) for y in range(0, 50, 5) for x in range(0, 50, 5)]
    if order == "reversed":
        pts = pts[::-1]
    elif order == "column_major":
        pts = [(x, y) for x in range(0, 50, 5) for y in range(0, 50, 5)]
    elif order.startswith("shuffled"):
        rng = np.random.default_rng(int(order[-1]))
        pts = [pts[i] for i in rng.permutation(len(pts))]
    assert len(check_same(shim, pts)) == 2 * 9 * 9


@pytest.mark.parametrize("case", ["extension_then_edges", "unsorted_chain", "apex_below", "vertical"])
def test_collinear_chain_then_points_on_its_extension_and_hull_edges(shim, case):
    if case == "extension_then_edges":
        # chain, apex, both extensions of the chain (collinear with a hull edge), then points on each hull edge
        pts = [(10, 10), (20, 10), (30, 10), (30, 20), (40, 10), (0, 10), (50, 10), (30, 15), (20, 15), (45, 5), (5, 10)]
    elif case == "unsorted_chain":           # the chain must be sorted before the fan
        pts = [(30, 10), (10, 10), (50, 10), (20, 10), (40, 10), (25, 30), (60, 10), (0, 10), (25, 20), (35, 20)]
    elif case == "apex_below":               # the first point off the chain on its right: the fan in the other order
        pts = [(10, 30), (40, 30), (20, 30), (30, 30), (25, 5), (50, 30), (0, 30), (25, 30 + 1), (45, 30), (30, 20)]
        pts = list(dict.fromkeys(pts))
    else:                                    # a vertical chain with points on its extension and between its points
        pts = [(7, 0), (7, 40), (7, 20), (20, 20), (7, 60), (7, 10), (7, 50), (0, 30), (13, 30), (7, 30)]
    assert len(check_same(shim, pts)) > 0


@pytest.mark.parametrize("seed,n", [(11, 2000), (12, 3000)])
def test_random_sets_equal_the_restatement(shim, seed, n):
    rng = np.random.default_rng(seed)
    pts = list(dict.fromkeys(tuple(map(int, p)) for p in rng.integers(0, 4097, size=(n, 2))))
    pts += [(0, 0), (4096, 4096), (0, 4096), (4096, 0)]
    pts = list(dict.fromkeys(pts))
    assert len(check_same(shim, pts)) > n


@pytest.mark.parametrize("keep", [1.0, 0.8, 0.5])
def test_lattices_to_the_coordinate_bound(shim, keep):
    """64-px lattices over 0..4096, whole and thinned: every quadrilateral cocircular, the predicates at their bound"""
    rng = np.random.default_rng(int(keep * 10))
    pts = [(x, y) for y in range(0, 4097, 64) for x in range(0, 4097, 64) if rng.random() < keep or keep == 1.0]
    tris = check_same(shim, pts)
    if keep == 1.0:
        assert len(tris) == 2 * 64 * 64


# ---- triangle planes --------------------------------------------------------------------------------------------------
def _camera(rng):
    f = rng.uniform(300, 3000)
    K = np.array([[f, 0, rng.uniform(0, 4096)], [0, f * rng.uniform(0.9, 1.1), rng.uniform(0, 4096)], [0, 0, 1]])
    return np.linalg.inv(K).astype(np.float32)


def _unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v)


def _plane_through(n, X):
    n = _unit(n)
    return np.array([*n, -n @ X], np.float32)


def _raw_cross(Kinv, xs, ys, planes):
    Ki = np.asarray(Kinv, np.float64).reshape(3, 3)
    X = []
    for i in range(3):
        r = Ki @ np.array([xs[i], ys[i], 1.0])
        p = np.asarray(planes[i], np.float64)
        X.append(-p[3] / (p[:3] @ r) * r)
    X = np.asarray(X)
    return np.cross(X[1] - X[0], X[2] - X[0]) @ X.sum(0)


def _same(shim, Kinv, xs, ys, planes):
    got = cpp_triangle_plane(shim, Kinv, xs, ys, planes)
    want = pyprior.triangle_plane(Kinv, xs, ys, np.asarray(planes, np.float32))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (got, want)
    return got


def test_triangle_planes_equal_the_restatement_on_random_triangles(shim):
    rng = np.random.default_rng(5)
    flipped = kept = 0
    for _ in range(400):
        Kinv = _camera(rng)
        xs, ys = rng.integers(0, 4097, 3), rng.integers(0, 4097, 3)
        planes = []
        for i in range(3):
            r = Kinv.astype(np.float64) @ np.array([xs[i], ys[i], 1.0])
            X = rng.uniform(0.5, 50.0) * r
            n = _unit(rng.normal(0, 1, 3))
            planes.append(_plane_through(n if n @ X < 0 else -n, X))
        got = _same(shim, Kinv, xs, ys, planes)
        if got.any():
            assert abs(np.linalg.norm(got[:3].astype(np.float64)) - 1.0) < 1e-6
        s = _raw_cross(Kinv, xs, ys, planes)
        flipped += s > 0
        kept += s < 0
    assert flipped > 50 and kept > 50                            # both branches of the orientation rule


def test_triangle_plane_zero_cross_product_is_all_zero(shim):
    rng = np.random.default_rng(6)
    Kinv = _camera(rng)
    xs, ys = [10, 400, 90], [20, 30, 700]
    zero_d = [np.array([*_unit(rng.normal(0, 1, 3)), 0.0], np.float32) for _ in range(3)]       # every point at the centre
    got = _same(shim, Kinv, xs, ys, zero_d)
    assert not got.view(np.uint32).any()
    # one shared plane at three collinear pixels: the points are collinear, the cross product exactly zero
    p = _plane_through([0.0, 0.0, -1.0], np.array([0.0, 0.0, 7.0]))
    got = _same(shim, Kinv, [0, 64, 128], [0, 0, 0], [p, p, p])
    assert not got.view(np.uint32).any()
    # a repeated vertex
    got = _same(shim, Kinv, [5, 5, 300], [9, 9, 40], [p, p, p])
    assert not got.view(np.uint32).any()


def test_triangle_plane_flips_towards_the_camera(shim):
    Kinv = np.linalg.inv(np.array([[800.0, 0, 320], [0, 800, 240], [0, 0, 1]])).astype(np.float32)
    p = _plane_through([0.1, -0.2, -1.0], np.array([0.0, 0.0, 5.0]))
    ccw = ([100, 500, 300], [100, 120, 400])
    cw = ([100, 300, 500], [100, 400, 120])
    assert _raw_cross(Kinv, *ccw, [p, p, p]) * _raw_cross(Kinv, *cw, [p, p, p]) < 0   # one of the two orders is flipped
    a = _same(shim, Kinv, *ccw, [p, p, p])
    b = _same(shim, Kinv, *cw, [p, p, p])
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert a[2] < 0 and a[3] > 0                                  # faces the camera: n.X0 < 0
    assert np.abs(a.astype(np.float64) - p.astype(np.float64)).max() < 1e-5


def test_triangle_plane_almost_parallel_to_a_ray(shim):
    rng = np.random.default_rng(8)
    for k in range(60):
        Kinv = _camera(rng)
        xs, ys = rng.integers(0, 4097, 3), rng.integers(0, 4097, 3)
        planes = []
        for i in range(3):
            r = _unit(Kinv.astype(np.float64) @ np.array([xs[i], ys[i], 1.0]))
            t = _unit(np.cross(r, rng.normal(0, 1, 3)))             # a normal perpendicular to the ray
            n = _unit(t + 10.0 ** -rng.uniform(3, 7) * r) if i == k % 3 else _unit(-r + 0.3 * t)
            planes.append(_plane_through(n, rng.uniform(1, 20) * r))
        _same(shim, Kinv, xs, ys, planes)

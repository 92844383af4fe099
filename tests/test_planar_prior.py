"""Planar prior (DESIGN.md §18) without a device: the term's known answers, the triangulation's empty-circle property and
agreement with scipy, the rasterisation's coverage, the planes of a sampled plane, the header's layout and the refusals
that happen before the library loads."""
from __future__ import annotations

import ctypes as C
import os
import re
import sys
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pyprior  # noqa: E402
from gipuma_b200 import api  # noqa: E402


def _cam(fx=500.0, fy=500.0, cx=40.0, cy=30.0):
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    return types.SimpleNamespace(K=K.ravel(), K_inv=np.linalg.inv(K.astype(np.float64)).astype(np.float32).ravel(),
                                 fx=np.float32(fx), alpha=np.float32(np.float32(fx) / np.float32(fy)))


# ---- the term -------------------------------------------------------------------------------------------------------
def test_term_known_answers():
    n = np.array([0.0, 0.0, -1.0, 5.0], np.float32)
    w, sd, ns = 0.5, 0.1, pyprior.normal_scale(5.0)
    assert pyprior.term(n, n, np.float32(5), np.float32(5), w, sd, ns) == 0.0
    far = pyprior.term(n, n, np.float32(1e6), np.float32(5), w, sd, ns)
    assert far == np.float32(w)
    nan = pyprior.term(n, n, np.float32(np.nan), np.float32(5), w, sd, ns)
    assert nan == np.float32(w)
    for d in (1e-3, 0.05, 0.3, 2.0):
        up = pyprior.term(n, n, np.float32(5 + d), np.float32(5), w, sd, ns)
        dn = pyprior.term(n, n, np.float32(5 - d), np.float32(5), w, sd, ns)
        delta_up = np.float32(np.float32(5 + d) - np.float32(5))
        delta_dn = np.float32(np.float32(5) - np.float32(5 - d))
        if delta_up == delta_dn:
            assert up == dn
        assert 0 < up < w
    # one sigma in depth: q = 1, the term is weight / 2
    assert pyprior.term(n, n, np.float32(5.25), np.float32(5), w, np.float32(0.25), ns) == np.float32(0.25)
    # normals: 0 for equal normals, grows with the angle, saturates
    tilt = [pyprior.term(np.array([np.sin(a), 0, -np.cos(a), 5], np.float32), n, np.float32(5), np.float32(5), w, sd, ns)
            for a in np.radians([0, 2, 5, 20, 90])]
    assert tilt[0] == 0 and all(a < b for a, b in zip(tilt, tilt[1:])) and tilt[-1] < w


def test_with_prior_keeps_maxcost_and_pixels_without_prior():
    cam = _cam()
    H, W = 6, 8
    planes = np.tile(np.array([0, 0, -1, 5], np.float32), (H, W, 1))
    pm = planes.copy()
    pm[:, :4] = 0.0                                            # left half: no prior
    pm[0, 5, 3] = 50.0                                         # depth -50: out of range, no prior
    cost = np.full((H, W), 0.3, np.float32)
    cost[1, 6] = pyprior.MAXCOST
    planes[2, 7, 3] = 5.5
    out = pyprior.with_prior(cost, planes, pm, cam, 1.0, 10.0, 0.5, 0.1, 5.0)
    assert (out[:, :4] == cost[:, :4]).all() and out[0, 5] == cost[0, 5] and out[1, 6] == pyprior.MAXCOST
    assert out[2, 7] > cost[2, 7] and out[3, 6] == cost[3, 6]


# ---- triangulation --------------------------------------------------------------------------------------------------
def _empty_circle(pts, tris):
    P = [tuple(map(int, p)) for p in pts]
    for a, b, c in tris:
        assert pyprior.orient(P[a], P[b], P[c]) > 0
        for d in range(len(P)):
            if d not in (a, b, c):
                assert pyprior.incircle(P[a], P[b], P[c], P[d]) <= 0, (a, b, c, d)


def _hull_area2(pts):
    from scipy.spatial import ConvexHull
    return 2 * ConvexHull(np.asarray(pts, float)).volume


def _area2(pts, tris):
    P = np.asarray(pts, np.int64)
    return sum(pyprior.orient(P[a], P[b], P[c]) for a, b, c in tris)


@pytest.mark.parametrize("seed,n", [(0, 30), (1, 200), (2, 500)])
def test_delaunay_random_sets(seed, n):
    rng = np.random.default_rng(seed)
    pts = {tuple(p) for p in rng.integers(0, 300, size=(n, 2))}
    pts = [p for p in pts]
    rng.shuffle(pts)
    tris = pyprior.delaunay(pts)
    _empty_circle(pts, tris)
    assert _area2(pts, tris) == round(_hull_area2(pts))


@pytest.mark.parametrize("kind", ["rows", "grid", "cocircular", "collinear_start", "border"])
def test_delaunay_degenerate_sets(kind):
    if kind == "rows":                       # collinear rows of points, row after row
        pts = [(x, y) for y in (0, 7, 14) for x in range(0, 60, 5)]
    elif kind == "grid":                     # every quadrilateral cocircular
        pts = [(x, y) for y in range(0, 50, 5) for x in range(0, 50, 5)]
    elif kind == "cocircular":               # squares and a regular octagon's lattice points on one circle
        pts = [(0, 0), (10, 0), (10, 10), (0, 10), (5, 5), (5, -5), (15, 5), (5, 15), (-5, 5), (8, 1), (2, 9)]
    elif kind == "collinear_start":          # many collinear points before the first that is not
        pts = [(x, 3) for x in range(0, 40, 3)] + [(17, 20), (4, 0), (33, 1), (20, -9)]
    else:                                    # support points of a 5 px grid hugging the image border
        rng = np.random.default_rng(7)
        pts = [(min(5 * cx + int(rng.integers(0, 2)) * 4, 61), 5 * cy + int(rng.integers(0, 5)))
               for cy in range(9) for cx in range(13)]
        pts = list(dict.fromkeys(pts))
    tris = pyprior.delaunay(pts)
    _empty_circle(pts, tris)
    assert _area2(pts, tris) == round(_hull_area2(pts))


def test_delaunay_fewer_than_three_or_collinear():
    assert len(pyprior.delaunay([])) == 0
    assert len(pyprior.delaunay([(1, 1), (2, 2)])) == 0
    assert len(pyprior.delaunay([(x, 2 * x) for x in range(10)])) == 0


def test_delaunay_equals_scipy_in_general_position():
    from scipy.spatial import Delaunay
    rng = np.random.default_rng(3)
    pts = [tuple(p) for p in {tuple(p) for p in rng.integers(0, 4096, size=(400, 2))}]
    tris = pyprior.delaunay(pts)
    ref = Delaunay(np.asarray(pts, float)).simplices
    canon = lambda t: tuple(sorted(map(int, t)))  # noqa: E731
    assert sorted(canon(t) for t in tris) == sorted(canon(t) for t in ref)


# ---- rasterisation --------------------------------------------------------------------------------------------------
def _inside_hull(pts, H, W):
    """strictly inside the convex hull / on its boundary, in exact integers"""
    from scipy.spatial import ConvexHull
    P = np.asarray(pts, np.int64)
    hv = P[ConvexHull(P.astype(float)).vertices]             # counter-clockwise in scipy's (x, y) frame
    ys, xs = np.mgrid[0:H, 0:W]
    o = [(hv[(i + 1) % len(hv), 0] - hv[i, 0]) * (ys - hv[i, 1]) - (hv[(i + 1) % len(hv), 1] - hv[i, 1]) * (xs - hv[i, 0])
         for i in range(len(hv))]
    o = np.stack(o)
    return (o > 0).all(0), (o >= 0).all(0)


@pytest.mark.parametrize("kind", ["random", "grid", "rows"])
def test_raster_exactly_once_inside_hull(kind):
    H, W = 60, 80
    rng = np.random.default_rng(5)
    if kind == "random":
        pts = list(dict.fromkeys(tuple(map(int, p)) for p in rng.integers(0, [W, H], size=(120, 2))))
    elif kind == "grid":
        pts = [(x, y) for y in range(0, H, 6) for x in range(0, W, 6)]
    else:
        pts = [(x, y) for y in range(2, H, 11) for x in range(1, W, 7)]
    tris = pyprior.delaunay(pts)
    _, count = pyprior.raster_cover(pts, tris, H, W)
    strict, closed = _inside_hull(pts, H, W)
    assert (count[strict] == 1).all()
    assert (count[~closed] == 0).all() and (count <= 1).all()


# ---- a known plane --------------------------------------------------------------------------------------------------
def test_support_of_a_plane_reproduces_it():
    cam = _cam(fx=300.0, fy=320.0, cx=41.5, cy=29.0)
    H, W = 60, 80
    n = np.array([0.2, -0.1, -1.0])
    n /= np.linalg.norm(n)
    X0 = np.array([0.0, 0.0, 6.0])
    d = -n @ X0
    planes = np.tile(np.array([*n, d], np.float32), (H, W, 1))
    rng = np.random.default_rng(0)
    cost = rng.random((H, W)).astype(np.float32)
    pts, tris, pm, counts = pyprior.build(planes, cost, 5, 2.0, cam, 1.0, 20.0)
    assert counts[0] == len(pts) == 12 * 16 and counts[1] == len(tris) > 0
    has, _ = pyprior.has_prior(pm, cam, 1.0, 20.0)
    assert counts[2] == has.sum() > 0.5 * H * W
    got = pm[has].astype(np.float64)
    assert np.abs(got[:, :3] - n).max() < 1e-5 and np.abs(got[:, 3] - d).max() < 1e-5 * abs(d)




# ---- the C-ABI structs and the refusals before the library loads ----------------------------------------------------
def test_structs_match_the_header():
    with open(os.path.join(ROOT, "include", "gipuma_b200.h")) as fh:
        h = fh.read()
    for name, cls in (("gpm_prior_build", api.GpmPriorBuild), ("gpm_prior_info", api.GpmPriorInfo)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), h, re.S).group(1)
        assert re.findall(r"^\s*[a-z ]+?\s+([a-z_]+);", body, re.M) == [f for f, _ in cls._fields_], name
    assert C.sizeof(api.GpmPriorBuild) == 8 and C.sizeof(api.GpmPriorInfo) == 24
    for fn in ("gpm_set_planar_prior", "gpm_get_planar_prior", "gpm_build_planar_prior", "gpm_set_prior", "gpm_offer_prior"):
        assert re.search(r"\bint %s\(gpm_ctx\* ctx" % fn, h), fn


@pytest.mark.parametrize("args", [(-1.0, 1.0, 5.0), (float("nan"), 1.0, 5.0), (float("inf"), 1.0, 5.0), (0.5, 0.0, 5.0),
                                  (0.5, float("inf"), 5.0), (0.5, 1.0, 0.0), (0.5, 1.0, 91.0), (0.5, 1.0, float("nan"))])
def test_prior_arguments_refused_before_the_library(args, monkeypatch):
    monkeypatch.setattr(api, "load_library", lambda: pytest.fail("library loaded"))
    with pytest.raises(ValueError):
        api.check_prior(*args)


@pytest.mark.parametrize("args", [(0, 1.0), (65, 1.0), (2.5, 1.0), (5, float("nan"))])
def test_build_arguments_refused_before_the_library(args, monkeypatch):
    monkeypatch.setattr(api, "load_library", lambda: pytest.fail("library loaded"))
    with pytest.raises(ValueError):
        api.check_prior_build(*args)
    api.check_prior_build(5, float("inf"))
    api.check_prior(0.0, 1.0, 5.0)

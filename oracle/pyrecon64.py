"""Float64 references of the fusion (DESIGN.md §12, §22) and the meshing (DESIGN.md §24), with a rounding bound on every
quantity the fp32 kernels compute.

TEST INFRASTRUCTURE: only tests/ may import this.  Unlike the C restatements, which repeat the kernels' fp32 operations
in the kernels' order, these are the same formulas in plain float64, so a formula that both the kernel and its
restatement got wrong would show here.

Rounding bound (a running error bound, derived, not tuned).  Every quantity q the kernels compute is carried here as a
pair (v, e): v its value in float64 from the same fp32 inputs, e a bound on |q_fp32 - v|.  Inputs are exact (e = 0).
An fp32 operation rounds to nearest: fl(a o b) = (a o b)(1 + d), |d| <= u = 2^-24, plus an absolute error of at most
2^-150 when the result is subnormal.  With |a_fp32 - a| <= ea and |b_fp32 - b| <= eb:

    add/sub   |fl(a' + b') - (a + b)|  <= ea + eb + u (|a + b| + ea + eb)
    mul       |fl(a' b') - a b|        <= |a| eb + |b| ea + ea eb + u (|a| + ea)(|b| + eb)
    div       |fl(a' / b') - a / b|    <= (ea + |a / b| eb) / (|b| - eb) + u (|a| + ea) / (|b| - eb)     (|b| > eb)
    sqrt      |fl(sqrt(a')) - sqrt(a)| <= max(sqrt(a + ea) - sqrt(a), sqrt(a) - sqrt(max(a - ea, 0)))
                                          + u sqrt(a + ea)

and float64's own rounding (2^-53 relative per operation) is covered by taking u = 2^-24 + 2^-52.  A decision
"q < T" (T an fp32 threshold, exact) is *certain* when |v - T| > e: then the fp32 kernel takes the branch float64 takes.
A projection floor(q + 0.5) is certain when q + 0.5 lies more than its e from every integer.  Where a decision is not
certain, only the restatements can say what the kernel does.
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24 + 2.0 ** -52
ETA = 2.0 ** -150


class R:
    """A float64 value with the bound of its fp32 counterpart's error (numpy arrays or scalars)."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v, self.e = np.broadcast_arrays(np.asarray(v, np.float64), np.asarray(e, np.float64))

    @staticmethod
    def of(x):
        return x if isinstance(x, R) else R(np.asarray(x, np.float64))

    def _round(self, v, e, mag):
        return R(v, e + U * mag + ETA)

    def __add__(self, o):
        o = R.of(o)
        v = self.v + o.v
        return self._round(v, self.e + o.e, np.abs(v) + self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = R.of(o)
        v = self.v - o.v
        return self._round(v, self.e + o.e, np.abs(v) + self.e + o.e)

    def __rsub__(self, o):
        return R.of(o) - self

    def __mul__(self, o):
        o = R.of(o)
        a, b = np.abs(self.v), np.abs(o.v)
        return self._round(self.v * o.v, a * o.e + b * self.e + self.e * o.e, (a + self.e) * (b + o.e))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = R.of(o)
        den = np.abs(o.v) - o.e
        with np.errstate(divide="ignore", invalid="ignore"):
            q = self.v / o.v
            e = np.where(den > 0, (self.e + np.abs(q) * o.e) / den, np.inf)
            mag = np.where(den > 0, (np.abs(self.v) + self.e) / den, np.inf)
        return self._round(q, e, mag)

    def __rtruediv__(self, o):
        return R.of(o) / self

    def __neg__(self):
        return R(-self.v, self.e)

    def __abs__(self):
        return R(np.abs(self.v), self.e)

    def sqrt(self):
        a = np.maximum(self.v, 0.0)
        s = np.sqrt(a)
        e = np.maximum(np.sqrt(a + self.e) - s, s - np.sqrt(np.maximum(a - self.e, 0.0)))
        return self._round(s, e, np.sqrt(a + self.e))

    def __getitem__(self, k):
        return R(self.v[k], self.e[k])


def less(q: R, t):
    """(q < t in float64, certain)"""
    return q.v < t, np.abs(q.v - t) > q.e


def greater(q: R, t):
    return q.v > t, np.abs(q.v - t) > q.e


def rounded(q: R):
    """(floor(q + 0.5), certain): the kernels' nearest pixel."""
    w = q + 0.5
    return np.floor(w.v), np.abs(w.v - np.round(w.v)) > w.e


def cameras(cams):
    """(M_inv [n, 3, 3], P [n, 3, 4], f [n]) float64 of the fusion's fp32 cameras (api.fuse_cameras)."""
    M = np.array([list(c.M_inv) for c in cams], np.float64).reshape(-1, 3, 3)
    P = np.array([list(c.P) for c in cams], np.float64).reshape(-1, 3, 4)
    f = np.array([c.f for c in cams], np.float64)
    return M, P, f


def _dot3(row, X):
    return ((R(row[0]) * X[0] + R(row[1]) * X[1]) + R(row[2]) * X[2])


def _project(P, X):
    return [_dot3(P[r, :3], X) + R(P[r, 3]) for r in range(3)]


def _backproject(M, P, x, y, d):
    """get3Dpoint: X = M_inv (d (x, y, 1) - P_col34)"""
    a, b, c = R(d) * x - R(P[0, 3]), R(d) * y - R(P[1, 3]), R(d) - R(P[2, 3])
    return [_dot3(M[i], (a, b, c)) for i in range(3)]


def fusion_decisions(norm4, cams, r, depth_min, depth_max, normal_thresh, rule="disparity", disp_thresh=0.1,
                     reproj_px=2.0, depth_rel=0.01):
    """The consistency test of every pixel of view r against every view j (DESIGN.md §12, §22), in float64.
    Returns dict: valid [npix] (the reference depth in range), ok [n, npix] (consistent; False for j = r), certain
    [n, npix] (the decision holds for the fp32 kernel), q [n, npix] (target pixel, -1 where there is none) and X (the
    reference point, 3 R)."""
    n4 = np.asarray(norm4, np.float32)
    n, H, W = n4.shape[:3]
    M, P, f = cameras(cams)
    nr = n4[r].reshape(-1, 4).astype(np.float64)
    p = np.arange(H * W)
    x, y, d = (p % W).astype(np.float64), (p // W).astype(np.float64), nr[:, 3]
    lo, hi = float(np.float32(depth_min)), float(np.float32(depth_max))
    valid = (d >= lo) & (d <= hi)
    X = _backproject(M[r], P[r], x, y, d)
    cos_t = float(np.float32(math.cos(float(np.float32(normal_thresh)) * math.pi / 180.0)))
    ok = np.zeros((n, H * W), bool)
    cert = np.ones((n, H * W), bool)
    qs = np.full((n, H * W), -1, np.int64)
    for j in range(n):
        if j == r:
            continue
        alive, sure = valid.copy(), np.ones(H * W, bool)

        def gate(passed, certain):
            nonlocal alive, sure
            sure &= ~alive | certain                           # a decision taken on a live path must be certain
            alive &= passed

        hx, hy, hz = _project(P[j], X)
        gate(*greater(hz, 0.0))
        with np.errstate(all="ignore"):
            fu, cu = rounded(hx / hz)
            fv, cv = rounded(hy / hz)
        gate(np.ones(H * W, bool), cu & cv)
        gate((fu >= 0) & (fu < W) & (fv >= 0) & (fv < H), np.ones(H * W, bool))
        with np.errstate(invalid="ignore"):
            q = np.where(alive, np.nan_to_num(fv * W + fu), 0).astype(np.int64)
        t = n4[j].reshape(-1, 4)[q].astype(np.float64)
        gate((t[:, 3] >= lo) & (t[:, 3] <= hi), np.ones(H * W, bool))
        with np.errstate(all="ignore"):
            if rule == "disparity":
                fb = R(f[j]) * float(np.float32(0.54))
                gate(*less(abs(fb / hz - fb / R(t[:, 3])), float(np.float32(disp_thresh))))
            else:
                Xj = _backproject(M[j], P[j], fu, fv, t[:, 3])
                gx, gy, gz = _project(P[r], Xj)
                gate(*greater(gz, 0.0))
                dx, dy = gx / gz - x, gy / gz - y
                gate(*less((dx * dx + dy * dy).sqrt(), float(np.float32(reproj_px))))
                gate(*less(abs(gz - d) / R(d), float(np.float32(depth_rel))))
            c = (R(nr[:, 0]) * t[:, 0] + R(nr[:, 1]) * t[:, 1]) + R(nr[:, 2]) * t[:, 2]
            gate(*greater(c, cos_t))
        ok[j], cert[j] = alive, sure
        qs[j] = np.where(alive, q, -1)
    return dict(valid=valid, ok=ok, certain=cert, q=qs, X=X)


def first_pass(norm4, cams, depth_min, depth_max, normal_thresh, num_consistent, images=None, **rule):
    """Pass 0 of the fusion (no marks exist yet) in float64: per pixel of view 0, whether it fuses, and its vertex.
    Returns dict: fused [npix], certain [npix] (every decision of the pixel certain), point / normal (3 R each: the mean
    point and the normalised normal sum), colour (3 R: the mean colour before clamping and rounding)."""
    n4 = np.asarray(norm4, np.float32)
    n, H, W = n4.shape[:3]
    dec = fusion_decisions(n4, cams, 0, depth_min, depth_max, normal_thresh, **rule)
    M, P, _ = cameras(cams)
    cnt = dec["ok"].sum(axis=0)
    fused = dec["valid"] & (cnt >= num_consistent)
    certain = dec["certain"].all(axis=0)
    nr = n4[0].reshape(-1, 4).astype(np.float64)
    s = list(dec["X"])
    sn = [R(nr[:, k]) for k in range(3)]
    img = None if images is None else np.asarray(images, np.float32).reshape(n, H * W, -1).astype(np.float64)
    col = [R(np.zeros(H * W)) + R(img[0, :, min(k, img.shape[2] - 1)]) for k in range(3)] if img is not None else None
    for j in range(1, n):
        okj, q = dec["ok"][j], np.maximum(dec["q"][j], 0)
        t = n4[j].reshape(-1, 4)[q].astype(np.float64)
        with np.errstate(all="ignore"):
            Xj = _backproject(M[j], P[j], (q % W).astype(np.float64), (q // W).astype(np.float64), t[:, 3])
        for k in range(3):
            s[k] = _where(okj, s[k] + Xj[k], s[k])
            sn[k] = _where(okj, sn[k] + t[:, k], sn[k])
            if col is not None:
                col[k] = _where(okj, col[k] + img[j, q, min(k, img.shape[2] - 1)], col[k])
    m = (cnt + 1).astype(np.float64)
    with np.errstate(all="ignore"):
        ln = (sn[0] * sn[0] + sn[1] * sn[1] + sn[2] * sn[2]).sqrt()
        out = dict(fused=fused, certain=certain, point=[sk / m for sk in s], normal=[snk / ln for snk in sn], len=ln,
                   colour=None if col is None else [ck / m for ck in col])
    return out


def _where(c, a: R, b: R):
    return R(np.where(c, a.v, b.v), np.where(c, a.e, b.e))


def centre(o, i, s):
    """origin + (i + 0.5) voxel, as the kernels compute a lattice coordinate"""
    return R(float(np.float32(o))) + (R(np.asarray(i, np.float64)) + 0.5) * float(np.float32(s))


def tsdf(depth, cams, origin, voxel, dims, trunc, depth_min, depth_max):
    """TSDF integration (DESIGN.md §24) in float64.  Returns (D as R [nz, ny, nx], Wt int [nz, ny, nx], certain
    [nz, ny, nx]: every decision of the voxel certain)."""
    dep = np.asarray(depth, np.float32)
    n, H, W = dep.shape
    _, P, _ = cameras(cams)
    nx, ny, nz = (int(a) for a in dims)
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    X = [centre(origin[0], i.ravel(), voxel), centre(origin[1], j.ravel(), voxel), centre(origin[2], k.ravel(), voxel)]
    T = float(np.float32(trunc))
    lo, hi = float(np.float32(depth_min)), float(np.float32(depth_max))
    S = R(np.zeros(X[0].v.shape))
    w = np.zeros(X[0].v.shape, np.int64)
    certain = np.ones(X[0].v.shape, bool)
    for v in range(n):
        alive, sure = np.ones(w.shape, bool), np.ones(w.shape, bool)

        def gate(passed, c):
            nonlocal alive, sure
            sure &= ~alive | c
            alive &= passed

        hx, hy, hz = _project(P[v], X)
        gate(*greater(hz, 0.0))
        with np.errstate(all="ignore"):
            fu, cu = rounded(hx / hz)
            fv, cv = rounded(hy / hz)
        gate(np.ones(w.shape, bool), cu & cv)
        gate((fu >= 0) & (fu < W) & (fv >= 0) & (fv < H), np.ones(w.shape, bool))
        with np.errstate(invalid="ignore"):
            q = np.where(alive, np.nan_to_num(fv * W + fu), 0).astype(np.int64)
        d = dep[v].reshape(-1)[q].astype(np.float64)
        with np.errstate(invalid="ignore"):
            gate((d > 0) & (d >= lo) & (d <= hi), np.ones(w.shape, bool))
        sdf = R(d) - hz
        behind, c = less(sdf, -T)
        gate(~behind, c)
        # min(sdf, trunc) moves by no more than sdf does: its bound is sdf's
        contrib = R(np.minimum(sdf.v, T), sdf.e) / T
        S = _where(alive, S + contrib, S)
        w += alive
        certain &= sure
    with np.errstate(all="ignore"):
        D = S / np.maximum(w, 1).astype(np.float64)
    D = R(np.where(w > 0, D.v, np.nan), np.where(w > 0, D.e, 0.0))
    shape = (nz, ny, nx)
    return R(D.v.reshape(shape), D.e.reshape(shape)), w.reshape(shape), certain.reshape(shape)


DIRS = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1)]     # x, y, z, x+y, x+z, y+z, x+y+z


def mesh_vertices(D, origin, voxel):
    """The marching-tetrahedra vertices of a volume whose points are all valid, in float64: one per lattice edge (p, p + e)
    of the seven Kuhn directions whose ends differ in inside (D < 0), in (point, direction) order, at
    x_p + t (x_q - x_p), t = D_p / (D_p - D_q).  Every such edge lies in a tetrahedron of a cube of the box.  Returns
    3 R [V]."""
    D = np.asarray(D, np.float32)
    nz, ny, nx = D.shape
    k, j, i = (a.ravel() for a in np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij"))
    pts, dirs = [], []
    for r, e in enumerate(DIRS):
        ok = (i + e[0] < nx) & (j + e[1] < ny) & (k + e[2] < nz)
        pi = np.nonzero(ok)[0]
        dp = D.ravel()[pi]
        dq = D[k[pi] + e[2], j[pi] + e[1], i[pi] + e[0]]
        cross = (dp < 0) != (dq < 0)
        pts.append(pi[cross])
        dirs.append(np.full(int(cross.sum()), r))
    pts, dirs = np.concatenate(pts), np.concatenate(dirs)
    order = np.lexsort((dirs, pts))
    pts, dirs = pts[order], dirs[order]
    e = np.array(DIRS)[dirs]
    dp = R(D.ravel()[pts].astype(np.float64))
    dq = R(D[k[pts] + e[:, 2], j[pts] + e[:, 1], i[pts] + e[:, 0]].astype(np.float64))
    t = dp / (dp - dq)
    out = []
    for ax, idx in enumerate((i, j, k)):
        xp = centre(origin[ax], idx[pts], voxel)
        xq = centre(origin[ax], idx[pts] + e[:, ax], voxel)
        out.append(xp + t * (xq - xp))
    return out


def _uchar_range(m: R):
    """The uchar colours floor(clamp(mean) + 0.5) can take, NaN -> 0, given the bound of the mean (and the rounding of the
    + 0.5, at most 2^-16 below 256)."""
    def uc(x):
        x = np.where(np.isnan(x), 0.0, np.clip(x, 0.0, 255.0))
        return np.floor(x + 0.5)
    slack = m.e + 2.0 ** -16
    return uc(m.v - slack), uc(m.v + slack)


def check_first_pass(ref, verts, src, W, images=False):
    """Pass 0 of a fusion (vertices, sources: the PLY records and (view, pixel) sources of the whole run) against
    first_pass: where all of a pixel's decisions are certain, fused or not agree; where it fuses, the point, normal and
    colour lie within their bounds.  Returns the number of certain pixels checked."""
    k = src[:, 0] == 0
    pix = src[k, 1]
    v = verts[k]
    got = np.zeros(len(ref["fused"]), bool)
    got[pix] = True
    c = ref["certain"]
    bad = np.nonzero(c & (got != ref["fused"]))[0]
    assert len(bad) == 0, "pixels %s: fused %s, float64 says %s" % (bad[:8], got[bad[:8]], ref["fused"][bad[:8]])
    sel = c[pix] & ref["fused"][pix]
    p = pix[sel]
    for ax, name in enumerate("xyz"):
        r = ref["point"][ax]
        err = np.abs(v[name][sel].astype(np.float64) - r.v[p])
        assert (err <= r.e[p]).all(), "%s: %g beyond its bound %g" % (name, err.max(), r.e[p][np.argmax(err - r.e[p])])
    ln = ref["len"]
    nz = ln.v[p] - ln.e[p] > 0
    for ax, name in enumerate(("nx", "ny", "nz")):
        r = ref["normal"][ax]
        err = np.abs(v[name][sel].astype(np.float64) - r.v[p])
        assert (err[nz] <= r.e[p][nz]).all(), "%s beyond its bound" % name
        assert (v[name][sel][ln.v[p] == 0] == 0).all(), "%s of a zero normal sum must be 0" % name
    if images:
        for ax, name in enumerate(("red", "green", "blue")):
            lo, hi = _uchar_range(ref["colour"][ax][p])
            g = v[name][sel].astype(np.float64)
            assert ((g >= lo) & (g <= hi)).all(), "%s outside its bound" % name
    return int(c.sum())


def check_tsdf(ref, D, Wt):
    """D, Wt of an integration against tsdf's (D, Wt, certain): where all of a voxel's decisions are certain, Wt is exact
    and D within its bound (NaN where Wt = 0).  Returns the number of certain voxels."""
    D64, W64, c = ref
    D, Wt = np.asarray(D, np.float32), np.asarray(Wt)
    assert np.array_equal(Wt[c].astype(np.int64), W64[c]), "Wt differs at a certain voxel"
    seen = c & (W64 > 0)
    assert np.isnan(D[c & (W64 == 0)]).all()
    err = np.abs(D[seen].astype(np.float64) - D64.v[seen])
    assert (err <= D64.e[seen]).all(), "D beyond its bound by %g" % (err - D64.e[seen]).max()
    return int(c.sum())


def check_mesh_vertices(D, origin, voxel, v):
    """Vertices of a mesh of an all-valid volume against mesh_vertices: the same count, each within its bound."""
    ref = mesh_vertices(D, origin, voxel)
    v = np.asarray(v, np.float32)
    assert len(v) == len(ref[0].v), "%d vertices, float64 has %d" % (len(v), len(ref[0].v))
    for ax in range(3):
        err = np.abs(v[:, ax].astype(np.float64) - ref[ax].v)
        assert (err <= ref[ax].e).all(), "axis %d beyond its bound by %g" % (ax, (err - ref[ax].e).max())
    return len(v)

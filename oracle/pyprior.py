"""The planar prior (DESIGN.md §18), restated in numpy: the term, the support points, the Delaunay triangulation, the
triangles' planes and the rasterised prior map, each bit for bit with the library.

TEST INFRASTRUCTURE: only tests/ and tools/ may import this.

The term and every depth it reads use IEEE round-to-nearest float32 multiply, add, subtract and divide with denormals
flushed to zero (the kernels' .rn.ftz operations), so float32 numpy with a flush after each operation reproduces them.
The triangulation is the library's incremental Lawson algorithm step for step (gpm_prior.cpp), with exact integer
predicates; the triangle planes are its float64 arithmetic in the same order.
"""
from __future__ import annotations

import math

import numpy as np

MAXCOST = np.float32(1000.0)
_TINY = np.float32(1.17549435e-38)


def _ftz(x):
    x = np.asarray(x, dtype=np.float32)
    return np.where(np.abs(x) < _TINY, np.float32(0.0) * x, x).astype(np.float32)


def _op(f, *a):
    with np.errstate(all="ignore"):
        return _ftz(f(*[_ftz(v) for v in a]))


def fadd(a, b): return _op(np.add, a, b)
def fsub(a, b): return _op(np.subtract, a, b)
def fmul(a, b): return _op(np.multiply, a, b)
def fdiv(a, b): return _op(np.divide, a, b)


def normal_scale(normal_sigma_deg: float) -> np.float32:
    """1 - cos(sigma_n) as the library rounds it: in double, then to float."""
    return np.float32(1.0 - math.cos(float(normal_sigma_deg) * math.pi / 180.0))


def prior_depth(planes, cam, xs, ys):
    """plane_depth's formula (gipuma.cu:694-705) in IEEE float32: -d fx / (nx (x - K2) + alpha (ny (y - K5)) + nz fx).
    cam: the reference camera (fx, alpha, K as gpm_camera holds them)."""
    K = np.asarray(cam.K, np.float32).ravel()
    fx, K2, K5 = np.float32(cam.fx), K[2], K[5]
    alpha = np.float32(cam.alpha)
    p = np.asarray(planes, np.float32)
    xs = np.asarray(xs, np.float32)
    ys = np.asarray(ys, np.float32)
    t = fadd(fadd(fmul(p[..., 0], fsub(xs, K2)), fmul(alpha, fmul(p[..., 1], fsub(ys, K5)))), fmul(p[..., 2], fx))
    return fdiv(fmul(p[..., 3], -fx), t)


def term(hyp, prior, hd, pd, weight, depth_sigma, nscale):
    """prior(p, h) = weight * q / (1 + q), q = ((hd - pd) / sigma_d)^2 + max(0, 1 - n_h . n_pi) / nscale; weight where q is
    not finite or >= 1e30.  hyp, prior: [..., 4] planes; hd, pd: their prior_depth at the pixel."""
    h = np.asarray(hyp, np.float32)
    pi = np.asarray(prior, np.float32)
    delta = fdiv(fsub(hd, pd), np.float32(depth_sigma))
    dot = fadd(fadd(fmul(h[..., 0], pi[..., 0]), fmul(h[..., 1], pi[..., 1])), fmul(h[..., 2], pi[..., 2]))
    off = fsub(np.float32(1.0), dot)
    with np.errstate(invalid="ignore"):
        a = fdiv(np.where(off > 0, off, np.float32(0.0)), np.float32(nscale))
        q = fadd(fmul(delta, delta), a)
        frac = np.where(q < np.float32(1e30), fdiv(q, fadd(np.float32(1.0), q)), np.float32(1.0))
    return fmul(np.float32(weight), frac)


def has_prior(prior_map, cam, depth_min, depth_max):
    """[H, W] pixels whose prior plane's prior_depth lies in [depth_min, depth_max], and those depths."""
    H, W = prior_map.shape[:2]
    ys, xs = np.mgrid[0:H, 0:W]
    pd = prior_depth(prior_map, cam, xs, ys)
    with np.errstate(invalid="ignore"):
        return (pd >= np.float32(depth_min)) & (pd <= np.float32(depth_max)), pd


def with_prior(cost, planes, prior_map, cam, depth_min, depth_max, weight, depth_sigma, normal_sigma_deg):
    """The cost of each pixel's plane in prior mode, from its cost without the prior: unchanged where it is MAXCOST or the
    pixel has no prior, fadd(cost, prior) elsewhere."""
    H, W = cost.shape
    ys, xs = np.mgrid[0:H, 0:W]
    has, pd = has_prior(prior_map, cam, depth_min, depth_max)
    hd = prior_depth(planes, cam, xs, ys)
    t = term(planes, prior_map, hd, pd, weight, depth_sigma, normal_scale(normal_sigma_deg))
    cost = np.asarray(cost, np.float32)
    return np.where(has & (cost != MAXCOST), fadd(cost, np.where(has, t, np.float32(0.0))), cost).astype(np.float32)


def support(planes, cost, step, support_cost, cam, depth_min, depth_max):
    """Support points in cell order: [(x, y)] and their planes [n, 4].  Per step x step cell, the pixel with the smallest
    cost (NaN never wins, a tie goes to the lower (y, x)), kept when its cost < support_cost and its depth is in range."""
    H, W = cost.shape
    pts, pls = [], []
    for cy in range((H + step - 1) // step):
        for cx in range((W + step - 1) // step):
            c = cost[cy * step:(cy + 1) * step, cx * step:(cx + 1) * step]
            if np.isnan(c).all():
                continue
            cc = np.where(np.isnan(c), np.inf, c)
            i = int(np.argmin(cc))                          # first minimum in row-major order: the lower (y, x)
            y, x = cy * step + i // c.shape[1], cx * step + i % c.shape[1]
            if not (cost[y, x] < np.float32(support_cost)):
                continue
            d = prior_depth(planes[y, x], cam, np.float32(x), np.float32(y))
            if d >= np.float32(depth_min) and d <= np.float32(depth_max):
                pts.append((x, y))
                pls.append(planes[y, x])
    return pts, np.asarray(pls, np.float32).reshape(-1, 4)


# ---- Delaunay triangulation: gpm_prior.cpp's algorithm, step for step ------------------------------------------------
def orient(a, b, c):
    return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])


def incircle(a, b, c, d):
    """> 0: d strictly inside the circle through the counter-clockwise a, b, c (exact integer determinant)."""
    adx, ady = a[0] - d[0], a[1] - d[1]
    bdx, bdy = b[0] - d[0], b[1] - d[1]
    cdx, cdy = c[0] - d[0], c[1] - d[1]
    return ((adx * adx + ady * ady) * (bdx * cdy - cdx * bdy) + (bdx * bdx + bdy * bdy) * (cdx * ady - adx * cdy) +
            (cdx * cdx + cdy * cdy) * (adx * bdy - bdx * ady))


class _Mesh:
    def __init__(self, pts):
        self.p = pts
        self.v = []          # [[a, b, c]] counter-clockwise
        self.n = []          # [[na, nb, nc]] across the edge opposite each vertex, -1 on the hull
        self.last = 0

    def o(self, a, b, c):
        return orient(self.p[a], self.p[b], self.p[c])

    def add(self, a, b, c, na, nb, nc):
        self.v.append([a, b, c])
        self.n.append([na, nb, nc])
        return len(self.v) - 1

    def relink(self, x, frm, to):
        if x < 0:
            return
        for k in range(3):
            if self.n[x][k] == frm:
                self.n[x][k] = to
                return

    def legalize(self, tris):
        stack = list(reversed(tris))
        while stack:
            ti = stack.pop()
            ui = self.n[ti][0]
            if ui < 0:
                continue
            T, TN, U, UN = list(self.v[ti]), list(self.n[ti]), list(self.v[ui]), list(self.n[ui])
            j = UN.index(ti)
            p, a, b, q = T[0], T[1], T[2], U[j]
            if incircle(self.p[p], self.p[a], self.p[b], self.p[q]) <= 0:
                continue
            nta, ntb, nua, nub = TN[1], TN[2], UN[(j + 2) % 3], UN[(j + 1) % 3]
            self.v[ti], self.n[ti] = [p, a, q], [nub, ui, ntb]
            self.v[ui], self.n[ui] = [p, q, b], [nua, nta, ti]
            self.relink(nta, ti, ui)
            self.relink(nub, ui, ti)
            stack.append(ui)
            stack.append(ti)

    def next_hull(self, ti, k):
        b = self.v[ti][(k + 2) % 3]
        cur = ti
        while True:
            e = (self.v[cur].index(b) + 2) % 3
            if self.n[cur][e] < 0:
                return (cur, e)
            cur = self.n[cur][e]

    def prev_hull(self, ti, k):
        a = self.v[ti][(k + 1) % 3]
        cur = ti
        while True:
            e = (self.v[cur].index(a) + 1) % 3
            if self.n[cur][e] < 0:
                return (cur, e)
            cur = self.n[cur][e]

    def sees(self, ti, k, p):
        return self.o(self.v[ti][(k + 1) % 3], self.v[ti][(k + 2) % 3], p) < 0

    def insert(self, p):
        cur, out, steps = self.last, -1, 0
        while True:
            steps += 1
            if steps > 4 * len(self.v) + 16:
                raise RuntimeError("Delaunay walk did not terminate")
            out = -1
            for k in range(3):
                if self.o(self.v[cur][(k + 1) % 3], self.v[cur][(k + 2) % 3], p) < 0:
                    out = k
                    break
            if out < 0 or self.n[cur][out] < 0:
                break
            cur = self.n[cur][out]
        if out >= 0:
            first = (cur, out)
            while True:
                pr = self.prev_hull(*first)
                if pr == (cur, out) or not self.sees(pr[0], pr[1], p):
                    break
                first = pr
            edges = [first]
            while True:
                nx = self.next_hull(*edges[-1])
                if nx == first or not self.sees(nx[0], nx[1], p):
                    break
                edges.append(nx)
            base = len(self.v)
            fresh = []
            for e, (te, ke) in enumerate(edges):
                a, b = self.v[te][(ke + 1) % 3], self.v[te][(ke + 2) % 3]
                prev = base + e - 1 if e > 0 else -1
                nxt = base + e + 1 if e + 1 < len(edges) else -1
                fresh.append(self.add(p, b, a, te, prev, nxt))
                self.n[te][ke] = fresh[-1]
            self.last = fresh[0]
            self.legalize(fresh)
            return
        T, TN = list(self.v[cur]), list(self.n[cur])
        zeros = [k for k in range(3) if self.o(T[(k + 1) % 3], T[(k + 2) % 3], p) == 0]
        if len(zeros) > 1:
            raise RuntimeError("Delaunay: duplicate point")
        self.last = cur
        if not zeros:
            a, b, c = T
            t1, t2 = len(self.v), len(self.v) + 1
            self.v[cur], self.n[cur] = [p, b, c], [TN[0], t1, t2]
            self.add(p, c, a, TN[1], t2, cur)
            self.add(p, a, b, TN[2], cur, t1)
            self.relink(TN[1], cur, t1)
            self.relink(TN[2], cur, t2)
            self.legalize([cur, t1, t2])
            return
        i = zeros[0]
        c, a, b = T[i], T[(i + 1) % 3], T[(i + 2) % 3]
        ui = TN[i]
        t1 = len(self.v)
        u1 = t1 + 1 if ui >= 0 else -1
        self.v[cur], self.n[cur] = [p, c, a], [TN[(i + 2) % 3], u1, t1]
        self.add(p, b, c, TN[(i + 1) % 3], cur, ui)
        self.relink(TN[(i + 1) % 3], cur, t1)
        if ui < 0:
            self.legalize([cur, t1])
            return
        U, UN = list(self.v[ui]), list(self.n[ui])
        j = UN.index(cur)
        d = U[j]
        self.v[ui], self.n[ui] = [p, d, b], [UN[(j + 2) % 3], t1, u1]
        self.add(p, a, d, UN[(j + 1) % 3], ui, cur)
        self.relink(UN[(j + 1) % 3], ui, u1)
        self.legalize([cur, t1, ui, u1])


def delaunay(pts):
    """Triangles [m, 3] of the points [(x, y)] (distinct integers), inserted in the given order: counter-clockwise index
    triples, each rotated to start at its smallest index, sorted.  Nothing is triangulated until three points are not
    collinear; the first such point is joined to the sorted collinear chain."""
    pts = [(int(x), int(y)) for x, y in pts]
    M = _Mesh(pts)
    chain = []
    for p in range(len(pts)):
        if M.v:
            M.insert(p)
            continue
        if len(chain) < 2 or M.o(chain[0], chain[1], p) == 0:
            chain.append(p)
            continue
        chain.sort(key=lambda u: pts[u])
        left = M.o(chain[0], chain[1], p) > 0
        m = len(chain) - 1
        for k in range(m):
            prev, nxt = (k - 1 if k > 0 else -1), (k + 1 if k + 1 < m else -1)
            if left:
                M.add(p, chain[k], chain[k + 1], -1, nxt, prev)
            else:
                M.add(p, chain[k + 1], chain[k], -1, prev, nxt)
        M.last = 0
    out = []
    for v in M.v:
        r = v.index(min(v))
        out.append((v[r], v[(r + 1) % 3], v[(r + 2) % 3]))
    return np.asarray(sorted(out), np.int64).reshape(-1, 3)


def triangle_plane(Kinv, xs, ys, planes):
    """gpm_prior.cpp's triangle_plane: float64, the same operation order, rounded to float32; zeros where degenerate."""
    Ki = [float(v) for v in np.asarray(Kinv, np.float32).ravel()]
    X = []
    for i in range(3):
        px, py = float(xs[i]), float(ys[i])
        r = [(Ki[3 * k] * px + Ki[3 * k + 1] * py) + Ki[3 * k + 2] for k in range(3)]
        nx, ny, nz, d = (float(v) for v in planes[i])
        z = -d / ((nx * r[0] + ny * r[1]) + nz * r[2])
        X.append([z * r[k] for k in range(3)])
    e1 = [X[1][k] - X[0][k] for k in range(3)]
    e2 = [X[2][k] - X[0][k] for k in range(3)]
    c = [e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]]
    ln = math.sqrt((c[0] * c[0] + c[1] * c[1]) + c[2] * c[2])
    if ln == 0.0:
        return np.zeros(4, np.float32)
    c = [v / ln for v in c]
    s = [(X[0][k] + X[1][k]) + X[2][k] for k in range(3)]
    if (c[0] * s[0] + c[1] * s[1]) + c[2] * s[2] > 0.0:
        c = [-v for v in c]
    d = -((c[0] * X[0][0] + c[1] * X[0][1]) + c[2] * X[0][2])
    return np.asarray([c[0], c[1], c[2], d], np.float32)


def top_left(ax, ay, bx, by):
    return by > ay or (by == ay and bx < ax)


def raster_cover(pts, tris, H, W):
    """[H, W] index of the triangle each pixel belongs to under the top-left rule (-1: none), and the number of
    triangles that claim each pixel."""
    owner = -np.ones((H, W), np.int64)
    count = np.zeros((H, W), np.int64)
    P = np.asarray(pts, np.int64).reshape(-1, 2)
    for t, (i0, i1, i2) in enumerate(tris):
        v = P[[i0, i1, i2]]
        x0, x1 = max(int(v[:, 0].min()), 0), min(int(v[:, 0].max()), W - 1)
        y0, y1 = max(int(v[:, 1].min()), 0), min(int(v[:, 1].max()), H - 1)
        ys, xs = np.mgrid[y0:y1 + 1, x0:x1 + 1]
        inside = np.ones(xs.shape, bool)
        for e in range(3):
            ax, ay = v[e]
            bx, by = v[(e + 1) % 3]
            o = (bx - ax) * (ys - ay) - (by - ay) * (xs - ax)
            inside &= (o > 0) | ((o == 0) & top_left(ax, ay, bx, by))
        count[y0:y1 + 1, x0:x1 + 1] += inside
        owner[y0:y1 + 1, x0:x1 + 1][inside] = t
    return owner, count


def build(planes, cost, step, support_cost, cam, depth_min, depth_max):
    """The library's gpm_build_planar_prior from a state: (support points, triangles, prior map [H, W, 4], counts).
    cam: the reference camera (fx, alpha, K, K_inv as gpm_camera holds them)."""
    H, W = cost.shape
    Kinv = np.asarray(cam.K_inv, np.float32)
    pts, pls = support(planes, cost, step, support_cost, cam, depth_min, depth_max)
    tris = delaunay(pts)
    tplanes = [triangle_plane(Kinv, [pts[i][0] for i in t], [pts[i][1] for i in t], pls[list(t)]) for t in tris]
    owner, _ = raster_cover(pts, tris, H, W)
    prior_map = np.zeros((H, W, 4), np.float32)
    if len(tris):
        tp = np.asarray(tplanes, np.float32)
        m = owner >= 0
        prior_map[m] = tp[owner[m]]
    has, _ = has_prior(prior_map, cam, depth_min, depth_max)
    prior_map[~has] = 0.0
    return pts, tris, prior_map, (len(pts), len(tris), int(has.sum()))

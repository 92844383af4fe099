"""Float32 restatement of ACMH's refinement (DESIGN.md §23): the draws, the five candidates and the in-order accept.

hash:       key(s, i, r) = mix(mix(mix(s) ^ i) ^ r), draw k = mix(key ^ k), mix = lowbias32; uint32 arithmetic throughout.
            s = (uint32)seed ^ (uint32)(seed >> 32) of the context's 64-bit seed, i = y * W + x, r the launch counter.
uniform:    xorwow_uniform's map of a word x to (0, 1]: fma(float(x), 2^-32, 2^-33).
candidates: (d_r, n), (d, n_r), (d_r, n_r), (d, n_t), (d_t, n) from the plane at the start of the refinement, every step one
            IEEE float32 operation in the kernel's order (acmh_candidate in gpm_kernels.cuh); the fused multiply-adds are
            rounded once, exactly (fma32).
accept:     candidates in order, each taken where its cost is strictly below the running cost.
"""
from __future__ import annotations

import numpy as np

N_CANDIDATES = 5
PI32 = np.float32(3.14159274)
TINY = np.float32(2.0 ** -126)


def _ftz(x):
    """Flush float32 subnormals to a signed zero, as the kernels' .ftz operations do."""
    x = np.asarray(x, dtype=np.float32)
    return np.where(np.abs(x) < TINY, np.copysign(np.float32(0.0), x), x).astype(np.float32)


def fmul(a, b):
    with np.errstate(all="ignore"):
        return _ftz(np.multiply(a, b, dtype=np.float32))


def fadd(a, b):
    with np.errstate(all="ignore"):
        return _ftz(np.add(a, b, dtype=np.float32))


def fsub(a, b):
    with np.errstate(all="ignore"):
        return _ftz(np.subtract(a, b, dtype=np.float32))


def fdiv(a, b):
    with np.errstate(all="ignore"):
        return _ftz(np.divide(a, b, dtype=np.float32))


def fsqrt(a):
    with np.errstate(all="ignore"):
        return _ftz(np.sqrt(np.asarray(a, dtype=np.float32)))


def fma32(a, b, c):
    """a * b + c rounded once to float32 (round to nearest even).  The product of two float32 is exact in float64; the sum
    is taken in float64 with its rounding error (TwoSum), which decides the rare sums that fall on a float32 midpoint."""
    a, b, c = (np.asarray(v, dtype=np.float32) for v in (a, b, c))
    with np.errstate(all="ignore"):
        p = a.astype(np.float64) * b.astype(np.float64)
        c64 = c.astype(np.float64)
        s = p + c64
        bb = s - p
        e = (p - (s - bb)) + (c64 - bb)
        r = s.astype(np.float32)
        r64 = r.astype(np.float64)
        other = np.nextafter(r, np.where(s > r64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
        mid = np.isfinite(s) & (r64 != s) & ((r64 + other.astype(np.float64)) * 0.5 == s) & (e != 0)
        toward_other = (other.astype(np.float64) > r64) == (e > 0)
        r = np.where(mid & toward_other, other, r)
    return _ftz(r)


def mix(x):
    """lowbias32 on uint32 arrays."""
    x = np.asarray(x, dtype=np.uint32).copy()
    x ^= x >> np.uint32(16)
    x *= np.uint32(0x7FEB352D)
    x ^= x >> np.uint32(15)
    x *= np.uint32(0x846CA68B)
    x ^= x >> np.uint32(16)
    return x


def seed32(seed: int) -> int:
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return (seed & 0xFFFFFFFF) ^ (seed >> 32)


def key(seed: int, i, r: int):
    """Key of pixel index i (array) in launch r for the 64-bit context seed."""
    s = mix(np.uint32(seed32(seed)))
    return mix(mix(s ^ np.asarray(i, dtype=np.uint32)) ^ np.uint32(r & 0xFFFFFFFF))


def uniform(word):
    """(0, 1] from a uint32 word, as xorwow_uniform maps it."""
    f = np.asarray(word, dtype=np.uint32).astype(np.float64).astype(np.float32)
    return fma32(f, np.float32(2.3283064365386963e-10), np.float32(1.1641532182693481e-10))


def draw(k_arr, k):
    return uniform(mix(k_arr ^ np.asarray(k, dtype=np.uint32)))


def _cam(cam):
    """The reference camera's float32 fields the kernels read (RefCam, from a gpm_camera / api.GpmCamera)."""
    f = lambda v: np.asarray(list(v) if not np.isscalar(v) else v, dtype=np.float32)
    K = f(cam.K)
    return {"M": f(cam.M_inv), "P34": f(cam.P_col34), "C": f(cam.C), "K2": K[2], "K5": K[5], "fx": np.float32(cam.fx),
            "alpha": np.float32(cam.alpha), "f": np.float32(cam.f), "baseline": np.float32(cam.baseline)}


def prior_depth(c, n, fpx, fpy):
    """Depth at the pixel of plane n (..., 4) in IEEE multiply, add and divide (prior_depth in gpm_device.cuh)."""
    t = fadd(fadd(fmul(n[..., 0], fsub(fpx, c["K2"])), fmul(c["alpha"], fmul(n[..., 1], fsub(fpy, c["K5"])))),
             fmul(n[..., 2], c["fx"]))
    return fdiv(fmul(n[..., 3], -c["fx"]), t)


def dot3(ax, ay, az, bx, by, bz):
    return fma32(az, bz, fma32(ax, bx, fmul(ay, by)))


def plane_d(c, nx, ny, nz, fpx, fpy, depth):
    M, P34 = c["M"], c["P34"]
    X = fma32(depth, fpx, -P34[0])
    Y = fma32(depth, fpy, -P34[1])
    Z = fsub(depth, P34[2])
    wx = fma32(M[2], Z, fma32(M[0], X, fmul(M[1], Y)))
    wy = fma32(M[5], Z, fma32(M[3], X, fmul(M[4], Y)))
    wz = fma32(M[8], Z, fma32(M[6], X, fmul(M[7], Y)))
    return -dot3(nx, ny, nz, wx, wy, wz)


def ray(c, fpx, fpy):
    """The ray through each pixel, view_vector's formula without the normalisation."""
    M, P34, C = c["M"], c["P34"], c["C"]
    a, b, e = fsub(fpx, P34[0]), fsub(fpy, P34[1]), fsub(np.float32(1.0), P34[2])
    return tuple(fsub(fma32(e, M[3 * i + 2], fma32(a, M[3 * i], fmul(b, M[3 * i + 1]))), C[i]) for i in range(3))


def face(c, nx, ny, nz, v):
    flip = dot3(nx, ny, nz, *v) > 0
    return tuple(np.where(flip, -t, t).astype(np.float32) for t in (nx, ny, nz))


def marsaglia(k_arr, first: int = 5):
    """Marsaglia's sphere sampler per pixel from draws first, first + 1, ...: pairs until a*a + b*b < 1.  Returns the
    normal's components and the number of pairs each pixel drew."""
    shape = np.shape(k_arr)
    a = np.zeros(shape, np.float32)
    b = np.zeros(shape, np.float32)
    s = np.zeros(shape, np.float32)
    pairs = np.zeros(shape, np.int64)
    todo = np.ones(shape, bool)
    k = first
    while todo.any():
        u = fma32(draw(k_arr, k), np.float32(2.0), np.float32(-1.0))
        v = fma32(draw(k_arr, k + 1), np.float32(2.0), np.float32(-1.0))
        sm = fma32(u, u, fmul(v, v))
        a = np.where(todo, u, a)
        b = np.where(todo, v, b)
        s = np.where(todo, sm, s)
        pairs += todo
        todo &= sm >= 1.0
        k += 2
    sq = fsqrt(fsub(np.float32(1.0), s))
    return fmul(fadd(a, a), sq), fmul(fadd(b, b), sq), fsub(np.float32(1.0), fadd(s, s)), pairs


def candidates(planes, cam, min_disp, max_disp, depth_min, depth_max, eps, seed, r, ys=None, xs=None, width=None):
    """The five candidates [5, ...shape, 4] of the refinement of `planes` [..., 4] at pixels (ys, xs) (default: every pixel
    of an [H, W, 4] map) in launch r, with the parameters as the context holds them (float32) and the camera as a
    gpm_camera (api.pack_camera of the reference camera)."""
    planes = np.asarray(planes, dtype=np.float32)
    if ys is None:
        H, W = planes.shape[:2]
        ys, xs = np.mgrid[0:H, 0:W]
        width = W
    ys, xs = np.asarray(ys), np.asarray(xs)
    c = _cam(cam)
    f32 = np.float32
    eps, min_disp, max_disp = f32(eps), f32(min_disp), f32(max_disp)
    depth_min, depth_max = f32(depth_min), f32(depth_max)
    fpx, fpy = xs.astype(np.float32), ys.astype(np.float32)
    k_arr = key(seed, (ys.astype(np.int64) * int(width) + xs).astype(np.uint32), r)
    n = planes
    d = prior_depth(c, n, fpx, fpy)
    v = ray(c, fpx, fpy)
    # d_t (draw 0)
    s = fma32(draw(k_arr, 0), f32(2.0), f32(-1.0))
    with np.errstate(invalid="ignore"):
        d_t = np.fmin(depth_max, np.fmax(depth_min, fmul(d, fma32(eps, s, f32(1.0))))).astype(np.float32)
    # n_t (draws 1..3)
    dn = fmul(eps, PI32)
    two = fadd(dn, dn)
    t = [fadd(n[..., i], fma32(draw(k_arr, 1 + i), two, -dn)) for i in range(3)]
    rs = fdiv(f32(1.0), fsqrt(fma32(t[2], t[2], fma32(t[0], t[0], fmul(t[1], t[1])))))
    n_t = face(c, fmul(t[0], rs), fmul(t[1], rs), fmul(t[2], rs), v)
    # d_r (draw 4)
    disp = fma32(fsub(max_disp, min_disp), draw(k_arr, 4), min_disp)
    d_r = fdiv(fmul(c["f"], c["baseline"]), disp)
    # n_r (draws 5, 6, ...)
    mx, my, mz, _ = marsaglia(k_arr)
    n_r = face(c, mx, my, mz, v)
    n0 = (n[..., 0], n[..., 1], n[..., 2])
    out = []
    for normal, depth in ((n0, d_r), (n_r, d), (n_r, d_r), (n_t, d), (n0, d_t)):
        w = plane_d(c, normal[0], normal[1], normal[2], fpx, fpy, depth)
        out.append(np.stack([normal[0], normal[1], normal[2], w], axis=-1).astype(np.float32))
    return np.stack(out)


def candidate_depths(planes, cam, min_disp, max_disp, depth_min, depth_max, eps, seed, r):
    """(d, d_r, d_t) per pixel of an [H, W, 4] map: the start depth and the two drawn depths."""
    planes = np.asarray(planes, dtype=np.float32)
    H, W = planes.shape[:2]
    ys, xs = np.mgrid[0:H, 0:W]
    c = _cam(cam)
    fpx, fpy = xs.astype(np.float32), ys.astype(np.float32)
    k_arr = key(seed, (ys * W + xs).astype(np.uint32), r)
    d = prior_depth(c, planes, fpx, fpy)
    s = fma32(draw(k_arr, 0), np.float32(2.0), np.float32(-1.0))
    with np.errstate(invalid="ignore"):
        d_t = np.fmin(np.float32(depth_max), np.fmax(np.float32(depth_min), fmul(d, fma32(np.float32(eps), s, np.float32(1.0)))))
    disp = fma32(fsub(np.float32(max_disp), np.float32(min_disp)), draw(k_arr, 4), np.float32(min_disp))
    return d, fdiv(fmul(c["f"], c["baseline"]), disp), d_t.astype(np.float32)


def accept(planes, cost, cand, cand_cost, where):
    """The in-order accept at the pixels `where` [H, W]: candidate j replaces the running plane and cost where
    cand_cost[j] < running cost.  Returns (planes, cost, changed), changed marking the pixels that took any candidate."""
    planes = np.array(planes, dtype=np.float32, copy=True)
    cost = np.array(cost, dtype=np.float32, copy=True)
    changed = np.zeros(cost.shape, bool)
    for j in range(len(cand)):
        with np.errstate(invalid="ignore"):
            take = where & (np.asarray(cand_cost[j], dtype=np.float32) < cost)
        planes = np.where(take[..., None], cand[j], planes)
        cost = np.where(take, cand_cost[j], cost).astype(np.float32)
        changed |= take
    return planes, cost, changed


# ---- under joint view selection (jvs_pixel<..., REFINE_ACMH> in gpm_kernels.cuh) -----------------------------------------
# The refinement follows the launch's propagation fold in the same pixel and reuses its view weights w, which the launch's
# candidates in E decided (oracle/pyjvs.py; E is empty in a launch without propagation bits, so w then holds w_keep for
# the remembered views and 0 for the others).  Each of the five candidates of the plane the fold ended with is scored
# sum_j w_j c_j / sum_j w_j over its own per-view row (the kernel's row 8), or by the combination rule where sum_j w_j = 0,
# and accepted in candidate order with strict <.  The new selected-views mask is the propagation's, {j : w_j > 0}.

def jvs_accept(w, planes, cost, cand, cand_rows, cand_fallback, where):
    """The refinement's accept under joint view selection.  w [H, W, V]: the launch's weights; planes, cost: the state
    after the launch's fold; cand [5, H, W, 4]; cand_rows [5, H, W, V] float32: each candidate's per-view costs (NCC, plus
    the geometric term where it is on); cand_fallback [5, H, W]: the combination rule's cost of each candidate.  Returns
    (planes, cost, changed) as accept()."""
    from oracle import pyjvs
    costs = [pyjvs.weighted(w, cand_rows[j], cand_fallback[j]) for j in range(len(cand))]
    return accept(planes, cost, cand, costs, where)


def jvs_expected(planes, cost, masks, colour, mask, rows_of, fallback_of, ref_cam, cam, min_disp, max_disp, depth_min,
                 depth_max, eps, seed, r, params, t, adaptive=False):
    """State after one joint-view-selection launch with ACMH's refinement (mask bits 0 / 1 / 2: close / far / refine, as
    gpm_phase takes them) of checkerboard colour `colour`: oracle.pyjvs.expected's propagation, then, with bit 2, the
    refinement of launch r (the context's refinement counter).  rows_of, fallback_of, ref_cam, params and t as
    pyjvs.expected takes them; cam the reference camera as a gpm_camera (api.pack_camera).  Returns (planes, cost, masks,
    ambiguous, refined), refined marking the pixels that took a refinement candidate."""
    from oracle import pyjvs
    det = {}
    p, c, m, amb = pyjvs.expected(planes, cost, masks, colour, mask & 3, rows_of, fallback_of, ref_cam, depth_min, depth_max,
                                  params, t, adaptive=adaptive, details=det)
    refined = np.zeros(c.shape, bool)
    if mask & 4:
        H, W = c.shape
        ys, xs = np.mgrid[0:H, 0:W]
        cand = candidates(p, cam, min_disp, max_disp, depth_min, depth_max, eps, seed, r)
        rows = np.stack([rows_of(np.ascontiguousarray(cand[j]))[1] for j in range(len(cand))])
        fb = np.stack([fallback_of(np.ascontiguousarray(cand[j])) for j in range(len(cand))])
        p, c, refined = jvs_accept(det["w"], p, c, cand, rows, fb, ((xs + ys) & 1) == colour)
    return p, c, m, amb, refined

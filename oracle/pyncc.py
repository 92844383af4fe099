"""The NCC photometric cost (DESIGN.md §15), restated in numpy.

TEST INFRASTRUCTURE: only tests/ and tools/ may import this.

ncc_cost() is the device's setup_window sums and ncc_cost (gpm_device.cuh) operation for operation: every step is one
float32 multiply, add, subtract, divide or square root, rounded to nearest, which numpy's float32 arithmetic reproduces bit
for bit, and the device's flush of denormal results to zero is applied after every step.  Sums run sequentially from +0 in
sample order.  Per-view costs are combined by oracle/pygeo.combine.

sample_views64() and ncc_cost64() are the float64 layer for general scenes: the window's samples, support weights and
source-view values computed in float64 with a software bilinear filter (the texture's clamp addressing), for comparisons
within a tolerance.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
_TINY = np.finfo(np.float32).tiny


def _ftz(x):
    """float32, with denormals flushed to a zero of the same sign (the device's .ftz arithmetic)."""
    x = np.asarray(x, dtype=f32)
    return np.where(np.abs(x) < _TINY, np.copysign(f32(0.0), x), x).astype(f32)


def _mul(a, b):
    return _ftz(_ftz(a) * _ftz(b))


def _add(a, b):
    return _ftz(_ftz(a) + _ftz(b))


def _sub(a, b):
    return _ftz(_ftz(a) - _ftz(b))


def _div(a, b):
    with np.errstate(all="ignore"):
        return _ftz(_ftz(a) / _ftz(b))


def window_sums(w, r):
    """Per pixel, independent of the hypothesis: W = sum w_s, Sr = sum a_s, Srr = sum a_s r_s with a_s = w_s r_s.
    w, r: [..., ns] float32 in sample order."""
    w, r = np.asarray(w, dtype=f32), np.asarray(r, dtype=f32)
    Ws = Sr = Srr = np.zeros(w.shape[:-1], dtype=f32)
    for s in range(w.shape[-1]):
        a = _mul(w[..., s], r[..., s])
        Ws, Sr, Srr = _add(Ws, w[..., s]), _add(Sr, a), _add(Srr, _mul(a, r[..., s]))
    return Ws, Sr, Srr


def view_sums(w, r, t):
    """Per hypothesis and view: St = sum w_s t_s, Stt = sum (w_s t_s) t_s, Srt = sum a_s t_s.  t: [..., ns] like w."""
    w, r, t = (np.asarray(x, dtype=f32) for x in (w, r, t))
    St = Stt = Srt = np.zeros(t.shape[:-1], dtype=f32)
    for s in range(t.shape[-1]):
        wt = _mul(w[..., s], t[..., s])
        a = _mul(w[..., s], r[..., s])
        St, Stt, Srt = _add(St, wt), _add(Stt, _mul(wt, t[..., s])), _add(Srt, _mul(a, t[..., s]))
    return St, Stt, Srt


def cost_from_sums(Ws, Sr, Srr, St, Stt, Srt, min_std):
    """1 - c / sqrt(v_r v_t) clamped to [0, 2]; 2 where !(W > 0), !(v_r >= min_std^2), !(v_t >= min_std^2) or NaN."""
    mr, mt = _div(Sr, Ws), _div(St, Ws)
    vr = _sub(_div(Srr, Ws), _mul(mr, mr))
    vt = _sub(_div(Stt, Ws), _mul(mt, mt))
    c = _sub(_div(Srt, Ws), _mul(mr, mt))
    s2 = _mul(f32(min_std), f32(min_std))
    with np.errstate(all="ignore"):
        x = _sub(f32(1.0), _div(c, _ftz(np.sqrt(_mul(vr, vt)))))
        flat = ~(Ws > 0) | ~(vr >= s2) | ~(vt >= s2) | np.isnan(x)
    return np.where(flat, f32(2.0), np.clip(x, f32(0.0), f32(2.0))).astype(f32)


def ncc_cost(w, r, t, min_std):
    """Cost of each view.  w, r: [..., ns] the support weights and the reference values of the window in sample order;
    t: [V, ..., ns] (or [..., ns] for one view) the source views' values at the samples.  Returns [V, ...] (or [...])."""
    Ws, Sr, Srr = window_sums(w, r)
    St, Stt, Srt = view_sums(w, r, t)
    return cost_from_sums(Ws, Sr, Srr, St, Stt, Srt, min_std)


# ---- float64 layer for general scenes -----------------------------------------------------------------------------------

def window_offsets(box):
    """(i, j) offsets of the samples of gpm_cost_eval's window, in sample order: stride 2, i (x) outer, j (y) inner."""
    rad = (box - 1) // 2
    return [(i, j) for i in range(-rad, rad + 1, 2) for j in range(-rad, rad + 1, 2)]


def bilinear(img, x, y):
    """Linear filtering of a [H, W] image at unnormalised texture coordinates (texel k's centre at k + 0.5), clamp
    addressing, in float64 (the texture unit quantises the weights to 8 bits; this does not)."""
    H, W = img.shape
    xb, yb = np.asarray(x, np.float64) - 0.5, np.asarray(y, np.float64) - 0.5
    x0, y0 = np.floor(xb), np.floor(yb)
    ax, ay = xb - x0, yb - y0

    def tex(yy, xx):
        return img[np.clip(yy, 0, H - 1).astype(np.int64), np.clip(xx, 0, W - 1).astype(np.int64)].astype(np.float64)
    return ((1 - ay) * ((1 - ax) * tex(y0, x0) + ax * tex(y0, x0 + 1)) +
            ay * ((1 - ax) * tex(y0 + 1, x0) + ax * tex(y0 + 1, x0 + 1)))


def sample_views64(ref_img, view_imgs, ref_cam, view_cams, planes, box, gamma):
    """float64 w [H, W, ns], r [H, W, ns] and t [V, H, W, ns] of every pixel's plane: r and the centre value from the
    replicate-padded reference image, w = exp(-|r - centre| / gamma), t_s = bilinear(view, H_v (x, y, 1)) at the sample's
    pixel (x, y) with H_v = K_v (R_v - t_v n^T / d) K_ref^-1, + 0.5 texel."""
    ref = np.asarray(ref_img, np.float64)
    H, W = ref.shape
    ys, xs = np.mgrid[0:H, 0:W]
    offs = window_offsets(box)
    r = np.stack([ref[np.clip(ys + j, 0, H - 1), np.clip(xs + i, 0, W - 1)] for i, j in offs], axis=-1)
    w = np.exp(-np.abs(r - ref[..., None]) / float(gamma))
    Ki = np.asarray(ref_cam.K_inv, np.float64).reshape(3, 3)
    n = np.asarray(planes, np.float64)
    ts = []
    for img, cam in zip(view_imgs, view_cams):
        K = np.asarray(cam.K, np.float64).reshape(3, 3)
        R = np.asarray(cam.R, np.float64).reshape(3, 3)
        tv = np.asarray(cam.t, np.float64).reshape(3)
        # H = K (R - t n^T / d) K^-1 per pixel
        A = R[None, None] - tv[None, None, :, None] * n[..., None, :3] / n[..., 3, None, None]
        Hm = np.einsum("ab,hwbc,cd->hwad", K, A, Ki)
        tvals = []
        for i, j in offs:
            p = np.stack([xs + i, ys + j, np.ones_like(xs)], axis=-1).astype(np.float64)
            q = np.einsum("hwab,hwb->hwa", Hm, p)
            tvals.append(bilinear(np.asarray(img), q[..., 0] / q[..., 2] + 0.5, q[..., 1] / q[..., 2] + 0.5))
        ts.append(np.stack(tvals, axis=-1))
    return w, r, np.stack(ts)


def ncc_cost64(w, r, t, min_std):
    """The cost of §15 in float64 (two-pass means, no cancellation): [V, H, W] from sample_views64's arrays."""
    Ws = w.sum(-1)
    mr = (w * r).sum(-1) / Ws
    mt = (w * t).sum(-1) / Ws
    vr = (w * (r - mr[..., None]) ** 2).sum(-1) / Ws
    vt = (w * (t - mt[..., None]) ** 2).sum(-1) / Ws
    c = (w * (r - mr[..., None]) * (t - mt[..., None])).sum(-1) / Ws
    s2 = float(min_std) ** 2
    with np.errstate(all="ignore"):
        x = 1.0 - c / np.sqrt(vr * vt)
    return np.where((vr >= s2) & (vt >= s2) & ~np.isnan(x), np.clip(x, 0.0, 2.0), 2.0)

"""The image pyramid and the joint bilateral upsampling of planes (DESIGN.md §19), restated in numpy float32.

TEST INFRASTRUCTURE: only tests/ and tools/ may import this.

downsample() is gpm_downsample and jbu() the kernel of gpm_upsample_planes, operation for operation and in the same order:
every step is one float32 multiply, add, subtract, divide or square root, rounded to nearest with denormals kept, which is
what numpy's float32 arithmetic does and what gpm_scale.cu is compiled to.  The spatial weights are computed in double and
rounded once, as the library's host code does.  Vectorised over pixels; the candidate loop (j outer, i inner) is the
summation order.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
MAX_RADIUS = 4


def _binomial(a, b, c):
    return (f32(0.25) * a + f32(0.5) * b) + f32(0.25) * c


def downsample(img):
    """One pyramid level of img [H, W] or [H, W, C]: [(H + 1) // 2, (W + 1) // 2(, C)] float32.  Coarse pixel (xc, yc) is
    the [1 2 1] / 4 average around fine pixel (2 xc, 2 yc), borders replicated, rows first."""
    a = np.asarray(img, dtype=f32)
    H, W = a.shape[:2]
    xs = 2 * np.arange((W + 1) // 2)
    ys = 2 * np.arange((H + 1) // 2)
    xl, xr = np.maximum(xs - 1, 0), np.minimum(xs + 1, W - 1)
    yl, yr = np.maximum(ys - 1, 0), np.minimum(ys + 1, H - 1)
    h = _binomial(a[:, xl], a[:, xs], a[:, xr])
    return _binomial(h[yl], h[ys], h[yr]).astype(f32)


def pyramid(img, levels):
    out = [np.asarray(img, dtype=f32)]
    for _ in range(levels - 1):
        out.append(downsample(out[-1]))
    return out


def spatial_table(sigma_space):
    """ws[by, bx, j + 4, i + 4] = fp32(exp(-((2 i - bx)^2 + (2 j - by)^2) / (2 sigma_space^2))), computed in double."""
    r = np.arange(-MAX_RADIUS, MAX_RADIUS + 1, dtype=np.float64)
    t = np.empty((2, 2, 2 * MAX_RADIUS + 1, 2 * MAX_RADIUS + 1), np.float64)
    s = float(sigma_space)
    for by in range(2):
        for bx in range(2):
            dx = 2 * r[None, :] - bx
            dy = 2 * r[:, None] - by
            t[by, bx] = np.exp(-(dx * dx + dy * dy) / (2.0 * s * s))
    return t.astype(f32)


def _dot3(a0, a1, a2, x, y, z):
    return (a0 * x + a1 * y) + a2 * z


def jbu(coarse, guide, K_inv, depth_min, depth_max, radius, sigma_space, sigma_range):
    """gpm_upsample_planes: (planes [H, W, 4], depth [H, W]) of the fine level from the coarse level's raw planes
    coarse [Hc, Wc, 4], guided by the fine reference image guide [H, W] (grey) or [H, W, 4] (x, y, z compared); K_inv: the
    fine reference camera's K^-1 (row-major 9 or 3x3)."""
    cp = np.asarray(coarse, dtype=f32)
    g = np.asarray(guide, dtype=f32)
    H, W = g.shape[:2]
    Hc, Wc = cp.shape[:2]
    assert (Hc, Wc) == ((H + 1) // 2, (W + 1) // 2)
    Ki = np.asarray(K_inv, dtype=f32).ravel()
    lo, hi = f32(depth_min), f32(depth_max)
    k = f32(1.0 / (float(sigma_range) * float(sigma_range)))
    ws = spatial_table(sigma_space)
    ys, xs = np.mgrid[0:H, 0:W]
    px, py, one = xs.astype(f32), ys.astype(f32), f32(1.0)
    rx, ry, rz = (_dot3(Ki[3 * r], Ki[3 * r + 1], Ki[3 * r + 2], px, py, one) for r in range(3))
    cx, cy = xs >> 1, ys >> 1
    wtab = ws[ys & 1, xs & 1]                                         # [H, W, 9, 9]
    colour = g.ndim == 3
    zero = np.zeros((H, W), f32)
    sw, swz, nx, ny, nz = zero.copy(), zero.copy(), zero.copy(), zero.copy(), zero.copy()
    with np.errstate(all="ignore"):
        for j in range(-radius, radius + 1):
            qy = cy + j
            for i in range(-radius, radius + 1):
                qx = cx + i
                inside = (qy >= 0) & (qy < Hc) & (qx >= 0) & (qx < Wc)
                qyc, qxc = np.clip(qy, 0, Hc - 1), np.clip(qx, 0, Wc - 1)
                n = cp[qyc, qxc]
                z = (-n[..., 3]) / _dot3(n[..., 0], n[..., 1], n[..., 2], rx, ry, rz)
                ok = inside & np.isfinite(z) & (z >= lo) & (z <= hi)
                gq = g[2 * qyc, 2 * qxc]
                if colour:
                    dx, dy, dz = (g[..., c] - gq[..., c] for c in range(3))
                    d2 = _dot3(dx, dy, dz, dx, dy, dz)
                else:
                    d = g - gq
                    d2 = d * d
                wr = one / (one + d2 * k)
                w = wtab[..., j + MAX_RADIUS, i + MAX_RADIUS] * wr
                sw = np.where(ok, sw + w, sw)
                swz = np.where(ok, swz + w * z, swz)
                nx = np.where(ok, nx + w * n[..., 0], nx)
                ny = np.where(ok, ny + w * n[..., 1], ny)
                nz = np.where(ok, nz + w * n[..., 2], nz)
        ln = np.sqrt(_dot3(nx, ny, nz, nx, ny, nz))
        good = (sw > 0) & (ln > 0)
        Z = swz / sw
        ox, oy, oz = nx / ln, ny / ln, nz / ln
        od = -_dot3(ox, oy, oz, Z * rx, Z * ry, Z * rz)
    planes = np.stack([ox, oy, oz, od], axis=-1).astype(f32)
    planes[~good] = cp[cy, cx][~good]
    depth = np.where(good, Z, f32(0)).astype(f32)
    return planes, depth

"""The geometric-consistency term (DESIGN.md §14) and the combination of per-view costs, restated in numpy.

TEST INFRASTRUCTURE: only tests/ and tools/ may import this.

geo_cost() is the device's geo_cost (gpm_device.cuh) operation for operation: every step is one float32 multiply, add,
subtract, divide or square root, rounded to nearest, which numpy's float32 arithmetic reproduces bit for bit (the device
flushes denormals to zero; no step of a camera-scale computation produces one).  combine() is pmCostMultiview_cu's rule
(combine_views in gpm_device.cuh) over given per-view costs; its last step multiplies by the device's approximate
reciprocal of the view count, which numpy does not reproduce, so the caller supplies those reciprocals.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
MAXCOST = f32(1000.0)


def _sum3(m, x, y, z):
    """(m0 x + m1 y) + m2 z, each operation rounded to float32."""
    return (m[0] * x + m[1] * y) + m[2] * z


def geo_cost(planes, ref_cam, view_cam, depth, weight, max_err, depth_min, depth_max):
    """g_j [H, W] float32 of source view j for every pixel's plane.

    planes [H, W, 4] float32 (n.xyz, d) in the reference frame; ref_cam: K and K_inv of the reference; view_cam: K, K_inv, R,
    t of view j as the context holds them (re-based on the reference); depth [H, W]: view j's depth map."""
    planes = np.asarray(planes, dtype=f32)
    depth = np.asarray(depth, dtype=f32)
    H, W = planes.shape[:2]
    ys, xs = np.mgrid[0:H, 0:W]
    px, py = xs.astype(f32), ys.astype(f32)
    one, half = f32(1.0), f32(0.5)
    nx, ny, nz, d = (planes[..., i] for i in range(4))
    Ki = np.asarray(ref_cam.K_inv, dtype=f32).ravel()
    Kr = np.asarray(ref_cam.K, dtype=f32).ravel()
    K = np.asarray(view_cam.K, dtype=f32).ravel()
    Kj = np.asarray(view_cam.K_inv, dtype=f32).ravel()
    R = np.asarray(view_cam.R, dtype=f32).ravel()
    t = np.asarray(view_cam.t, dtype=f32).ravel()
    w_, m_ = f32(weight), f32(max_err)
    far = w_ * m_
    with np.errstate(all="ignore"):
        rx, ry, rz = _sum3(Ki[0:3], px, py, one), _sum3(Ki[3:6], px, py, one), _sum3(Ki[6:9], px, py, one)
        z = (-d) / ((nx * rx + ny * ry) + nz * rz)
        ok = z > 0
        X, Y, Z = z * rx, z * ry, z * rz
        xj = _sum3(R[0:3], X, Y, Z) + t[0]
        yj = _sum3(R[3:6], X, Y, Z) + t[1]
        zj = _sum3(R[6:9], X, Y, Z) + t[2]
        ok &= zj > 0
        qz = _sum3(K[6:9], xj, yj, zj)
        u = np.floor(_sum3(K[0:3], xj, yj, zj) / qz + half)
        v = np.floor(_sum3(K[3:6], xj, yj, zj) / qz + half)
        ok &= (u >= 0) & (u <= f32(W - 1)) & (v >= 0) & (v <= f32(H - 1))
        iu, iv = np.where(ok, u, 0).astype(np.int64), np.where(ok, v, 0).astype(np.int64)
        D = depth[iv, iu]
        ok &= (D > 0) & (D >= f32(depth_min)) & (D <= f32(depth_max))
        ax = D * _sum3(Kj[0:3], u, v, one) - t[0]
        ay = D * _sum3(Kj[3:6], u, v, one) - t[1]
        az = D * _sum3(Kj[6:9], u, v, one) - t[2]
        bx = (R[0] * ax + R[3] * ay) + R[6] * az
        by = (R[1] * ax + R[4] * ay) + R[7] * az
        bz = (R[2] * ax + R[5] * ay) + R[8] * az
        ok &= bz > 0
        pz = _sum3(Kr[6:9], bx, by, bz)
        ex = _sum3(Kr[0:3], bx, by, bz) / pz - px
        ey = _sum3(Kr[3:6], bx, by, bz) / pz - py
        err = np.sqrt(ex * ex + ey * ey)
        g = w_ * np.where(err < m_, err, m_)
    return np.where(ok, g, far).astype(f32)


def num_considered(costs, cost_comb, n_best):
    """How many of the sorted view costs the combination averages, per pixel: numConsidered of gipuma.cu:779-797."""
    costs = np.asarray(costs, dtype=f32)
    valid = (costs < MAXCOST).sum(axis=0)
    if cost_comb == 1:
        return np.minimum(valid, n_best)
    if cost_comb == 3:
        return np.full(valid.shape, costs.shape[0])
    return valid


def combine_sum(costs, cost_comb, n_best, good_factor):
    """The sum the combination divides: per pixel, the num_considered smallest of min(cost_j, MAXCOST) in ascending order
    (COMB_GOOD: each capped at good_factor times the smallest), added in float32.  costs: [V, H, W] float32."""
    c = np.minimum(np.asarray(costs, dtype=f32), MAXCOST)
    c = np.sort(c, axis=0)
    k = num_considered(costs, cost_comb, n_best)
    thresh = c[0] * f32(good_factor)
    s = np.zeros(c.shape[1:], dtype=f32)
    for i in range(c.shape[0]):
        ci = np.minimum(thresh, c[i]) if cost_comb == 3 else c[i]
        s = np.where(i < k, s + ci, s).astype(f32)
    return s, k


def combine(costs, cost_comb, n_best, good_factor, rcp):
    """combine_views: rcp[k] * sum over the k considered views; MAXCOST where k = 0 or the result is NaN, negative or above
    MAXCOST.  rcp: {k: the device's float32 reciprocal of k}; pixels whose k has no entry are NaN."""
    s, k = combine_sum(costs, cost_comb, n_best, good_factor)
    r = np.full(s.shape, np.nan, dtype=f32)
    for kk, val in rcp.items():
        r[k == kk] = f32(val)
    with np.errstate(invalid="ignore"):
        out = (r * s).astype(f32)
        bad = (k < 1) | (out > MAXCOST) | (out < 0)
    out[bad] = MAXCOST
    out[(k >= 1) & np.isnan(r)] = np.nan
    return out

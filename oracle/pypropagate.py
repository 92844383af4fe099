"""The acceptance rule of one propagation launch, restated in numpy.

TEST INFRASTRUCTURE: only tests/ and tools/ may import this.

A propagation launch of one checkerboard colour is a pure function of the planes and costs it starts from: a pixel of
colour c reads only planes of the other colour, cost(p, plane) is pure, and a candidate is accepted when its depth at the
pixel lies in [depthMin, depthMax] and its cost is strictly below the running cost (spatialPropagation_cu,
gipuma.cu:829-871), the candidates being offered in a fixed order.  So the state after the launch follows from the costs
of the neighbour-shifted plane maps, C_k = cost_of(shifted_k, site_k), folded in that order.  This holds at any image
size and whatever memo, provenance or identity history the implementation keeps.

The one step numpy cannot reproduce bit for bit is the depth-range test (the GPU's plane_depth uses an approximate
reciprocal).  Pixels where some offered candidate's depth lies within a narrow band of a bound are reported as
`ambiguous` and must be left out of a bit-exact comparison.
"""
from __future__ import annotations

import numpy as np

# Close (1 px) then far (5 px) candidates, each in the order up, down, left, right (gipuma.cu:1571-1582 close,
# :1450-1462 far) as (dy, dx); a candidate is offered when py > d-1, py < H-d, px > d-1, px < W-d respectively.
CLOSE = [(-1, 0), (1, 0), (0, -1), (0, 1)]
FAR = [(-5, 0), (5, 0), (0, -5), (0, 5)]

# The 20 candidates of the fused kernel gipuma_checkerboard_cu in source order (gipuma.cu:1236-1330: up 1/3/5, down
# 1/3/5 :1236-1264, left 1/3/5, right 1/3/5 :1266-1292, the four (±1, ±2) points :1295-1311, the four (±2, ±1) points
# :1312-1329) as (dy, dx), with that code's own guards written as margins (gx0, gx1, gy0, gy1): offered when
# px >= gx0, px <= W-1-gx1, py >= gy0, py <= H-1-gy1.  They are not the tightest guards: the (-2, ±1) points need
# py > 2, not py > 1.
FUSED = [
    ((-1, 0), (0, 0, 1, 0)), ((-3, 0), (0, 0, 3, 0)), ((-5, 0), (0, 0, 5, 0)),
    ((1, 0), (0, 0, 0, 1)), ((3, 0), (0, 0, 0, 3)), ((5, 0), (0, 0, 0, 5)),
    ((0, -1), (1, 0, 0, 0)), ((0, -3), (3, 0, 0, 0)), ((0, -5), (5, 0, 0, 0)),
    ((0, 1), (0, 1, 0, 0)), ((0, 3), (0, 3, 0, 0)), ((0, 5), (0, 5, 0, 0)),
    ((-1, 2), (0, 2, 1, 0)), ((1, 2), (0, 2, 0, 1)), ((-1, -2), (2, 0, 1, 0)), ((1, -2), (2, 0, 0, 1)),
    ((-2, -1), (1, 0, 3, 0)), ((-2, 1), (0, 1, 3, 0)), ((2, -1), (1, 0, 0, 2)), ((2, 1), (0, 1, 0, 2)),
]

# Rounding variant (gpm_cost_eval's "cost_variant") of each call site of the fused kernel: 20 candidates, then the
# refinement.  The same tables as GPM_FUSED_SITES_FLOAT / GPM_FUSED_SITES_FLOAT4 in gpm_device.cuh.
FUSED_SITES_FLOAT = (1, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1)
FUSED_SITES_FLOAT4 = (0, 0, 0, 0, 0, 0, 0, 0, 0, 9, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1)

# Relative half-width of the ambiguous band around depthMin / depthMax: 1e-5, widened where the denominator of the depth
# cancels.  The GPU's float32 plane_depth rounds five times in the denominator and three times after it (one of them the
# approximate reciprocal), so its relative error stays below 6 * 2^-24 * (cond + 1), cond = sum|terms| / |sum of terms|;
# the band allows 16 * 2^-24 * (cond + 1).
DEPTH_BAND = 1e-5


def propagation_site(k: int, fused: bool, color_images: bool) -> int:
    """cost_variant that reproduces the rounding of candidate k's cost: x-first (1) for float images and y-first (0) for
    float4 images in the separate close / far kernels; the call-site table in the fused kernel."""
    if fused:
        return (FUSED_SITES_FLOAT4 if color_images else FUSED_SITES_FLOAT)[k]
    return 0 if color_images else 1


def refine_site(fused: bool, color_images: bool) -> int:
    """cost_variant of the refinement's evaluations: 0 in the separate kernels, site 20 in the fused one."""
    return (FUSED_SITES_FLOAT4 if color_images else FUSED_SITES_FLOAT)[20] if fused else 0


def candidates(H: int, W: int, mask: int, fused: bool = False):
    """[(k, dy, dx, offered[H, W])] of one launch in the order the kernel folds them.  `mask` as gpm_phase takes it
    (bit 0 close, bit 1 far; in a fused context bit 0 selects the 20 fused candidates), or bit 3 for the 20 fused
    candidates as gpo_phase takes it."""
    ys, xs = np.mgrid[0:H, 0:W]
    out = []
    if fused or (mask & 8):
        if (mask & 8) or (fused and (mask & 1)):
            for k, ((dy, dx), (gx0, gx1, gy0, gy1)) in enumerate(FUSED):
                ok = (xs >= gx0) & (xs <= W - 1 - gx1) & (ys >= gy0) & (ys <= H - 1 - gy1)
                out.append((k, dy, dx, ok))
        return out
    for bit, table in ((1, CLOSE), (2, FAR)):
        if not (mask & bit):
            continue
        for j, (dy, dx) in enumerate(table):
            d = max(abs(dy), abs(dx))
            ok = [ys > d - 1, ys < H - d, xs > d - 1, xs < W - d][j]
            out.append((4 * (bit - 1) + j, dy, dx, ok))
    return out


def shifted(planes: np.ndarray, dy: int, dx: int, offered: np.ndarray) -> np.ndarray:
    """The plane map whose pixel p holds the plane of p + (dy, dx) where that candidate is offered, its own plane elsewhere."""
    s = np.roll(planes, shift=(-dy, -dx), axis=(0, 1))
    return np.ascontiguousarray(np.where(offered[..., None], s, planes), dtype=np.float32)


def depth64(planes: np.ndarray, cam):
    """Depth along the ray of every pixel of each pixel's plane, in float64, from the formula of plane_depth
    (getDepthFromPlane3_cu, gipuma.cu:694-705; gipuma_oracle.c:119-123), and the condition number of its denominator."""
    H, W = planes.shape[:2]
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    p = planes.astype(np.float64)
    fx, alpha = float(np.float32(cam.fx)), float(np.float32(cam.alpha))
    K = np.asarray(cam.K, dtype=np.float32).ravel().astype(np.float64)
    terms = (p[..., 0] * (xs - K[2]), p[..., 1] * (ys - K[5]) * alpha, p[..., 2] * fx)
    t = terms[0] + terms[1] + terms[2]
    with np.errstate(divide="ignore", invalid="ignore"):
        depth = -p[..., 3] * fx / t
        cond = (np.abs(terms[0]) + np.abs(terms[1]) + np.abs(terms[2])) / np.abs(t)
    depth = np.where(np.isnan(p[..., 3]), 1000.0, depth)                    # plane_depth's NaN guard
    return depth, np.where(np.isfinite(cond), np.maximum(cond, 1.0), np.inf)


def expected(planes, cost, colour, mask, cost_of, ref_cam, depth_min, depth_max, fused=False, color_images=False):
    """State after one propagation launch of checkerboard colour `colour` (0 = black: (x + y) even).

    planes [H, W, 4], cost [H, W] float32: the state before the launch.  cost_of(planes, site) -> [H, W] float32 is the
    cost of each pixel's plane with the rounding variant `site` (e.g. ctx.cost_eval under option cost_variant = site, or
    the oracle's cost_eval, which has one variant).  ref_cam: the reference camera (fx, alpha, K).
    Returns (planes, cost, ambiguous): pixels of the other colour unchanged; `ambiguous` marks the pixels of this colour
    where some offered candidate's depth lies within DEPTH_BAND (relative; wider where the depth's denominator cancels) of
    depth_min or depth_max, where the range test may go either way."""
    planes = np.ascontiguousarray(planes, dtype=np.float32)
    cost = np.ascontiguousarray(cost, dtype=np.float32)
    H, W = cost.shape
    ys, xs = np.mgrid[0:H, 0:W]
    mine = ((xs + ys) & 1) == colour
    lo, hi = float(np.float32(depth_min)), float(np.float32(depth_max))
    out_p, out_c = planes.copy(), cost.copy()
    ambiguous = np.zeros((H, W), bool)
    for k, dy, dx, ok in candidates(H, W, mask, fused):
        offered = ok & mine
        if not offered.any():
            continue
        cand = shifted(planes, dy, dx, offered)
        depth, cond = depth64(cand, ref_cam)
        with np.errstate(invalid="ignore"):
            band = np.maximum(DEPTH_BAND, 2.0 ** -20 * (cond + 1.0))
            near = (np.abs(depth - lo) <= band * abs(lo)) | (np.abs(depth - hi) <= band * abs(hi))
            in_range = (depth >= lo) & (depth <= hi)
        ambiguous |= offered & near
        c = np.asarray(cost_of(cand, propagation_site(k, fused or bool(mask & 8), color_images)), dtype=np.float32)
        accept = offered & in_range & (c < out_c)
        out_c = np.where(accept, c, out_c)
        out_p = np.where(accept[..., None], cand, out_p)
    return out_p, out_c, ambiguous

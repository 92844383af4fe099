"""Adaptive checkerboard sampling (DESIGN.md §16) restated in numpy: the region table, the choice of each direction's
candidate, and the state after one propagation launch in that mode.

TEST INFRASTRUCTURE: only tests/ and tools/ may import this.

Adaptive sampling (ACMH, Xu & Tao, CVPR 2019) keeps the sweep's 8 directions and its accept rule; it only changes which
plane direction k offers: the plane of the pixel with the lowest stored cost inside region k, by the costs the launch
starts from.  Region pixels are of the other checkerboard colour, whose planes and costs a launch never writes, so a
launch stays a pure function of its start state and the fold of oracle/pypropagate.py applies unchanged, with each
candidate plane map gathered from the chosen pixels instead of a fixed shift.
"""
from __future__ import annotations

import numpy as np

from oracle import pypropagate as pp

# Regions as (dy, dx) offsets, each in its scan order (the order that breaks ties), in the sweep's fold order: near up,
# down, left, right (V shapes reaching 4 px), then far up, down, left, right (axial strips at 3, 5, .., 23 px).
NEAR_UP = [(-1, 0), (-2, -1), (-2, 1), (-3, -2), (-3, 2), (-4, -3), (-4, 3)]
FAR_UP = [(-a, 0) for a in range(3, 24, 2)]


def _four(up):
    down = [(-dy, dx) for dy, dx in up]
    left = [(dx, dy) for dy, dx in up]                      # transposed: up's "along" axis becomes x
    right = [(dy, -dx) for dy, dx in left]
    return [up, down, left, right]


REGIONS = _four(NEAR_UP) + _four(FAR_UP)


def choose(cost: np.ndarray, H: int, W: int, mask: int):
    """[(k, src_y [H, W], src_x [H, W], offered [H, W])] of one launch in fold order.  Pixel p's candidate of direction k
    is the region pixel inside the image with the smallest cost (NaN counts as +inf, a tie goes to the earliest offset);
    it is offered when some region pixel lies inside the image and the launch's phase bit is set (`mask` as gpm_phase
    takes it: bit 0 near, bit 1 far).  Where nothing is offered src is p itself."""
    cost = np.asarray(cost, dtype=np.float32)
    key = np.where(np.isnan(cost), np.float32(np.inf), cost)
    ys, xs = np.mgrid[0:H, 0:W]
    out = []
    for k, region in enumerate(REGIONS):
        if not (mask >> (k >> 2)) & 1:
            continue
        best = np.full((H, W), np.inf, np.float32)
        found = np.zeros((H, W), bool)
        sy, sx = ys.copy(), xs.copy()
        for dy, dx in region:
            y, x = ys + dy, xs + dx
            inside = (y >= 0) & (y < H) & (x >= 0) & (x < W)
            c = key[np.clip(y, 0, H - 1), np.clip(x, 0, W - 1)]
            take = inside & (~found | (c < best))
            best = np.where(take, c, best)
            sy, sx = np.where(take, y, sy), np.where(take, x, sx)
            found |= inside
        out.append((k, sy, sx, found))
    return out


def expected(planes, cost, colour, mask, cost_of, ref_cam, depth_min, depth_max, color_images=False, adaptive=True):
    """State after one propagation launch of checkerboard colour `colour`, as oracle.pypropagate.expected (same arguments
    and result) for the 8-neighbour sweep; adaptive=True offers each direction's region choice (choose) instead of the
    fixed neighbour.  Rounding sites are the fixed mode's: x-first for grey images, y-first for colour ones."""
    if not adaptive:
        return pp.expected(planes, cost, colour, mask, cost_of, ref_cam, depth_min, depth_max, color_images=color_images)
    planes = np.ascontiguousarray(planes, dtype=np.float32)
    cost = np.ascontiguousarray(cost, dtype=np.float32)
    H, W = cost.shape
    ys, xs = np.mgrid[0:H, 0:W]
    mine = ((xs + ys) & 1) == colour
    lo, hi = float(np.float32(depth_min)), float(np.float32(depth_max))
    out_p, out_c = planes.copy(), cost.copy()
    ambiguous = np.zeros((H, W), bool)
    for k, sy, sx, ok in choose(cost, H, W, mask):
        offered = ok & mine
        if not offered.any():
            continue
        cand = np.ascontiguousarray(np.where(offered[..., None], planes[sy, sx], planes), dtype=np.float32)
        depth, cond = pp.depth64(cand, ref_cam)
        with np.errstate(invalid="ignore"):
            band = np.maximum(pp.DEPTH_BAND, 2.0 ** -20 * (cond + 1.0))
            near = (np.abs(depth - lo) <= band * abs(lo)) | (np.abs(depth - hi) <= band * abs(hi))
            in_range = (depth >= lo) & (depth <= hi)
        ambiguous |= offered & near
        c = np.asarray(cost_of(cand, pp.propagation_site(k, False, color_images)), dtype=np.float32)
        accept = offered & in_range & (c < out_c)
        out_c = np.where(accept, c, out_c)
        out_p = np.where(accept[..., None], cand, out_p)
    return out_p, out_c, ambiguous

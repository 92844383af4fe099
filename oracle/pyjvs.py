"""Joint view selection (DESIGN.md §17) restated in float32 numpy: the good threshold, the view weights, the weighted
cost and the state after one propagation launch in that mode.

TEST INFRASTRUCTURE: only tests/ and tools/ may import this.

Joint view selection (ACMH, Xu & Tao, CVPR 2019) keeps the sweep's candidates, range test and accept rule.  What changes
is the cost: per pixel and launch, the per-view NCC costs m[k][j] of the candidates k in E (offered and in the depth
range, duplicates once per occurrence) decide one weight per view, and every hypothesis of the pixel, the current plane
included, is scored with those weights.  The per-view rows are inputs here (the device's, e.g. from one-view contexts'
gpm_cost_eval), so every step below is a float32 operation numpy reproduces bit for bit, except the confidence's ex2,
which is exact only where its argument is 0 (beta = 1e30 makes kb = -0 and every confidence 1).
"""
from __future__ import annotations

import math

import numpy as np

from oracle import pyacs
from oracle import pypropagate as pp

f32 = np.float32
LOG2E = 1.4426950408889634
DEFAULTS = {"tau_init": 0.8, "alpha": 90.0, "tau_bad": 1.2, "n_good": 3, "n_bad": 3, "beta": 0.3, "w_keep": 0.2}


def tau_t(tau_init: float, alpha: float, t: int) -> np.float32:
    """The good threshold at iteration t: tau_init * exp(-t^2 / alpha) in double from the float32 parameters, rounded once."""
    return f32(float(f32(tau_init)) * math.exp(-float(t) * float(t) / float(f32(alpha))))


def kb(beta: float) -> np.float32:
    """-log2(e) / (2 beta^2) in double from the float32 beta, rounded once: conf(m) = ex2(m * m * kb)."""
    b = float(f32(beta))
    return f32(-LOG2E / (2.0 * b * b))


def conf(m, kb_):
    """ex2(fmul(fmul(m, m), kb)), the ex2 in float64 rounded to float32 (the device's MUFU.EX2 agrees exactly at 0)."""
    x = (np.asarray(m, f32) * np.asarray(m, f32)).astype(f32) * f32(kb_)
    return np.exp2(x.astype(f32).astype(np.float64)).astype(f32)


def mask_bits(masks, V: int):
    """[..., V] bool of uint64 selected-views masks."""
    m = np.asarray(masks, np.uint64)
    return ((m[..., None] >> np.arange(V, dtype=np.uint64)) & np.uint64(1)).astype(bool)


def pack_mask(sel):
    """uint64 masks of [..., V] bool."""
    sel = np.asarray(sel, bool)
    out = np.zeros(sel.shape[:-1], np.uint64)
    for j in range(sel.shape[-1]):
        out |= sel[..., j].astype(np.uint64) << np.uint64(j)
    return out


def weights(rows, in_e, remembered, params, t: int):
    """View weights of §17 steps 2 and 3.  rows: [K, ..., V] float32 photometric costs of the candidates in fold order;
    in_e: [K, ...] bool, candidate k is in E; remembered: [..., V] bool, the pixel's mask.  Returns w [..., V] float32."""
    p = dict(DEFAULTS, **params)
    tt, kb_, tb = tau_t(p["tau_init"], p["alpha"], t), kb(p["beta"]), f32(p["tau_bad"])
    rows = np.asarray(rows, f32)
    good = np.zeros(rows.shape[1:], np.int64)
    bad = np.zeros(rows.shape[1:], np.int64)
    s = np.zeros(rows.shape[1:], f32)
    for k in range(rows.shape[0]):
        m, e = rows[k], np.asarray(in_e[k], bool)[..., None]
        g = e & (m < tt)
        good += g
        bad += e & (m > tb)
        s = np.where(g, (s + conf(m, kb_)).astype(f32), s)
    with np.errstate(divide="ignore", invalid="ignore"):
        rule = (s / good.astype(f32)).astype(f32)
    keep = np.asarray(remembered, bool) & (bad < p["n_bad"])
    w = np.where((good >= p["n_good"]) & (bad < p["n_bad"]), rule, np.where(keep, f32(p["w_keep"]), f32(0.0)))
    return w.astype(f32)


def weighted(w, c, fallback):
    """§17 step 4: sum_j w_j c_j / sum_j w_j, both sums sequential in ascending j from +0; `fallback` (the combination
    rule's cost of the same hypothesis) where sum_j w_j = 0.  w, c: [..., V] float32."""
    w, c = np.asarray(w, f32), np.asarray(c, f32)
    num = np.zeros(w.shape[:-1], f32)
    den = np.zeros(w.shape[:-1], f32)
    for j in range(w.shape[-1]):
        num = (num + (w[..., j] * c[..., j]).astype(f32)).astype(f32)
        den = (den + w[..., j]).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        out = (num / den).astype(f32)
    return np.where(den == 0, np.asarray(fallback, f32), out).astype(f32)


def candidate_maps(planes, cost, colour, mask, adaptive):
    """[(k, candidate plane map, offered [H, W])] of one launch in fold order, offered only at this colour's pixels:
    oracle/pyacs.py's choice when adaptive, oracle/pypropagate.py's fixed neighbours otherwise."""
    H, W = cost.shape
    ys, xs = np.mgrid[0:H, 0:W]
    mine = ((xs + ys) & 1) == colour
    out = []
    if adaptive:
        for k, sy, sx, ok in pyacs.choose(cost, H, W, mask):
            offered = ok & mine
            out.append((k, np.ascontiguousarray(np.where(offered[..., None], planes[sy, sx], planes), dtype=f32), offered))
    else:
        for k, dy, dx, ok in pp.candidates(H, W, mask):
            offered = ok & mine
            out.append((k, pp.shifted(planes, dy, dx, offered), offered))
    return out


def expected(planes, cost, masks, colour, mask, rows_of, fallback_of, ref_cam, depth_min, depth_max, params, t: int,
             adaptive: bool = False, details: dict = None):
    """State after one propagation launch (mask bits 0 / 1: close / far, as gpm_phase takes them) of checkerboard colour
    `colour` with joint view selection at iteration count t.

    planes [H, W, 4], cost [H, W] float32, masks [H, W] uint64: the state before the launch.  rows_of(planes) -> (m, c),
    each [H, W, V] float32: every pixel's per-view photometric costs of its plane, and the costs the weights multiply
    (m, or m + g with the geometric term).  fallback_of(planes) -> [H, W] float32: the combination rule's cost of each
    pixel's plane (today's NCC cost).  Returns (planes, cost, masks, ambiguous) as oracle.pypropagate.expected, the
    other colour unchanged.  `details`, if given, receives the weights "w" [H, W, V], the re-scored current cost "start"
    and the candidates' costs "scores" [K, H, W] in fold order, +inf where a candidate is not in E."""
    planes = np.ascontiguousarray(planes, dtype=f32)
    cost = np.ascontiguousarray(cost, dtype=f32)
    masks = np.asarray(masks, np.uint64)
    H, W = cost.shape
    ys, xs = np.mgrid[0:H, 0:W]
    mine = ((xs + ys) & 1) == colour
    lo, hi = float(f32(depth_min)), float(f32(depth_max))
    ambiguous = np.zeros((H, W), bool)
    cands = []
    for k, cand, offered in candidate_maps(planes, cost, colour, mask, adaptive):
        if not offered.any():
            continue
        depth, cond = pp.depth64(cand, ref_cam)
        with np.errstate(invalid="ignore"):
            band = np.maximum(pp.DEPTH_BAND, 2.0 ** -20 * (cond + 1.0))
            near = (np.abs(depth - lo) <= band * abs(lo)) | (np.abs(depth - hi) <= band * abs(hi))
            in_range = (depth >= lo) & (depth <= hi)
        ambiguous |= offered & near
        m, c = rows_of(cand)
        cands.append((cand, offered & in_range, m, c, fallback_of(cand)))
    m0, c0 = rows_of(planes)
    V = m0.shape[-1]
    if cands:
        w = weights(np.stack([x[2] for x in cands]), np.stack([x[1] for x in cands]), mask_bits(masks, V), params, t)
    else:
        w = weights(np.zeros((0, H, W, V), f32), np.zeros((0, H, W), bool), mask_bits(masks, V), params, t)
    out_c = weighted(w, c0, fallback_of(planes))
    out_p = planes.copy()
    if details is not None:
        details.update(w=w, start=out_c.copy(), scores=[])
    for cand, e, m, c, fb in cands:
        ck = weighted(w, c, fb)
        if details is not None:
            details["scores"].append(np.where(e, ck, f32(np.inf)))
        accept = e & (ck < out_c)
        out_c = np.where(accept, ck, out_c)
        out_p = np.where(accept[..., None], cand, out_p)
    out_m = np.where(mine, pack_mask(w > 0), masks)
    return (np.where(mine[..., None], out_p, planes).astype(f32), np.where(mine, out_c, cost).astype(f32), out_m,
            ambiguous)

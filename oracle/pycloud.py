"""Restatements of the nearest-neighbour distance of gpm_nearest_dist (DESIGN.md §13), the checker of the GPU search.

TEST INFRASTRUCTURE: only tests/ and tools/ may import this.

brute():     the specification evaluated over every pair, numpy float32 in the same operation order.  numpy neither fuses
             nor reorders elementwise operations, so this is exact by construction.
certified(): for large sets.  scipy's cKDTree gives each query's k + 1 nearest neighbours in float64; d2 is recomputed in
             float32 for the first k and the minimum kept.  A query is certified when no other data point can have a smaller
             float32 d2: the (k + 1)-th float64 distance, lowered by the fp32 error bound of d2, is at least that minimum (or
             at least the smallest d2 whose root exceeds max_dist, beyond which every result is +inf).  Uncertified queries
             go to brute().
"""
from __future__ import annotations

import numpy as np

INF = np.float32(np.inf)


def sqrt_threshold(max_dist) -> np.float32:
    """The smallest float32 v with sqrt(v) > max_dist (float32, correctly rounded): every d2 >= v gives +inf."""
    m = np.float32(max_dist)
    v = np.float32(m * m)
    if np.sqrt(v) > m:
        while v > 0 and np.sqrt(np.nextafter(v, np.float32(0))) > m:
            v = np.nextafter(v, np.float32(0))
    else:
        while not np.sqrt(v) > m:
            v = np.nextafter(v, INF)
    return np.float32(v)


def _finish(m, max_dist):
    D = np.sqrt(m.astype(np.float32))
    return np.where(D <= np.float32(max_dist), D, INF).astype(np.float32)


def brute_d2(query, data, block: int = 1 << 22) -> np.ndarray:
    """min over the data of fl32((dx*dx + dy*dy) + dz*dz) for every query (+inf for empty data)."""
    q = np.ascontiguousarray(query, dtype=np.float32).reshape(-1, 3)
    b = np.ascontiguousarray(data, dtype=np.float32).reshape(-1, 3)
    m = np.full(len(q), INF, dtype=np.float32)
    if len(b) == 0:
        return m
    rows = max(1, block // len(b))
    bx, by, bz = b[:, 0][None, :], b[:, 1][None, :], b[:, 2][None, :]
    for s in range(0, len(q), rows):
        qq = q[s:s + rows]
        dx = qq[:, 0:1] - bx
        dy = qq[:, 1:2] - by
        dz = qq[:, 2:3] - bz
        d2 = (dx * dx + dy * dy) + dz * dz
        m[s:s + rows] = d2.min(axis=1)
    return m


def brute(query, data, max_dist) -> np.ndarray:
    return _finish(brute_d2(query, data), max_dist)


def certified(query, data, max_dist, k: int = 8, workers: int = -1):
    """Returns (dist float32, certified bool per query before the brute-force fallback)."""
    from scipy.spatial import cKDTree
    q = np.ascontiguousarray(query, dtype=np.float32).reshape(-1, 3)
    b = np.ascontiguousarray(data, dtype=np.float32).reshape(-1, 3)
    if len(b) == 0 or len(q) == 0:
        return np.full(len(q), INF, dtype=np.float32), np.ones(len(q), dtype=bool)
    vstar = np.float64(sqrt_threshold(max_dist))
    # beyond this float64 radius every point's fp32 d2 is >= vstar (DESIGN.md §13): those neighbours need not be listed
    bound = float(max_dist) * (1.0 + 1e-5)
    kk = min(k + 1, len(b))
    dist, idx = cKDTree(b.astype(np.float64)).query(q.astype(np.float64), k=kk, distance_upper_bound=bound, workers=workers)
    dist, idx = dist.reshape(len(q), kk), idx.reshape(len(q), kk)
    m = np.full(len(q), INF, dtype=np.float32)
    for j in range(min(k, kk)):
        ok = idx[:, j] < len(b)
        c = b[np.where(ok, idx[:, j], 0)]
        dx, dy, dz = q[:, 0] - c[:, 0], q[:, 1] - c[:, 1], q[:, 2] - c[:, 2]
        d2 = (dx * dx + dy * dy) + dz * dz
        m = np.where(ok, np.minimum(m, d2), m)
    if kk <= k:                                               # every data point is a candidate
        nxt = np.full(len(q), np.inf)
    else:
        nxt = np.where(np.isinf(dist[:, k]), bound, dist[:, k])
    # fl32(d2) >= D^2 (1 - 5u) - 2^-148 for a true distance D; 1e-6 also covers the float64 error of cKDTree's distances
    lb = nxt * nxt * (1.0 - 1e-6) - 1e-44
    cert = lb >= np.minimum(m.astype(np.float64), vstar)
    out = _finish(m, max_dist)
    if not cert.all():
        out[~cert] = brute(q[~cert], b, max_dist)
    return out, cert

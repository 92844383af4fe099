"""Float32 restatement of the detail restorer's host steps and of the masked geometric cost (DESIGN.md §21).

detect:      pixel p is a detail pixel where fsub(c_ms[p], c_ph[p]) > threshold, one float32 rounding; NaN never is.
merge:       the photometric-only plane at detail pixels, the geometric stage's plane elsewhere ([H, W, 4], y then x).
masked_cost: the cost with the geometric term's mask is, per pixel, the cost with the term off where the mask is set and
             the cost with the term on elsewhere.
"""
from __future__ import annotations

import numpy as np


def detect(c_ms, c_ph, threshold) -> np.ndarray:
    """Detail mask [H, W] uint8 of the two photometric cost maps."""
    c_ms = np.asarray(c_ms, dtype=np.float32)
    c_ph = np.asarray(c_ph, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        diff = np.subtract(c_ms, c_ph, dtype=np.float32)
        return (diff > np.float32(threshold)).astype(np.uint8)


def merge(planes_ms, planes_ph, detail) -> np.ndarray:
    """Merged planes [H, W, 4]: planes_ph where detail is set, planes_ms elsewhere."""
    planes_ms = np.asarray(planes_ms, dtype=np.float32)
    planes_ph = np.asarray(planes_ph, dtype=np.float32)
    return np.where(np.asarray(detail)[..., None] != 0, planes_ph, planes_ms).astype(np.float32)


def masked_cost(cost_geo_on, cost_geo_off, mask) -> np.ndarray:
    """Per-pixel select: cost_geo_off where mask is nonzero, cost_geo_on elsewhere."""
    return np.where(np.asarray(mask) != 0, np.asarray(cost_geo_off, np.float32), np.asarray(cost_geo_on, np.float32))

"""ctypes binding of oracle/libfusion_rule_oracle.so — the scalar C restatement of the depth-map fusion under either
consistency rule (fusion_rule_oracle.c; DESIGN.md §22).

TEST INFRASTRUCTURE: only tests/, __graft_entry__ and tools/ may import this.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "libfusion_rule_oracle.so")
RULES = {"disparity": 0, "reprojection": 1}                   # GPM_FUSE_DISPARITY, GPM_FUSE_REPROJECTION


def build(force: bool = False) -> str:
    srcs = [os.path.join(_HERE, f) for f in ("fusion_rule_oracle.c", "fusion_oracle.c")]
    hdr = os.path.join(os.path.dirname(_HERE), "include", "gipuma_b200.h")
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in srcs + [hdr]):
        base = ["gcc", "-O2", "-fPIC", "-shared", "-fno-fast-math", "-ffp-contract=off", "-o", LIB, srcs[0], "-lm"]
        # OpenMP over the rows of a pass's candidate step where the toolchain has libgomp; scalar otherwise
        if subprocess.call(base[:2] + ["-fopenmp"] + base[2:], stderr=subprocess.DEVNULL) != 0:
            subprocess.check_call(base)
    return LIB


def fuse(norm4, cams, depth_min, depth_max, disp_thresh, normal_thresh, num_consistent, images=None, refs=None, used=None,
         threads: int = 1, rule: str = "disparity", reproj_px: float = 2.0, depth_rel: float = 0.01):
    """oracle.pyfusion.fuse under `rule`: "disparity" (disp_thresh) or "reprojection" (reproj_px, depth_rel; disp_thresh
    is not read).  Returns (vertices as api.PLY_VERTEX records, sources [count, 2] int32, used [n, H, W] uint8)."""
    from gipuma_b200.api import PLY_VERTEX
    lib = C.CDLL(build())
    n4 = np.ascontiguousarray(norm4, dtype=np.float32)
    n, H, W = n4.shape[:3]
    img = None if images is None else np.ascontiguousarray(images, dtype=np.float32)
    ch = 0 if img is None else (4 if img.ndim == 4 else 1)
    u = np.zeros((n, H, W), np.uint8) if used is None else np.array(used, dtype=np.uint8, order="C", copy=True)
    r0, r1 = (0, n) if refs is None else refs
    d = n4[r0:r1, ..., 3]
    cap = int(((d >= np.float32(depth_min)) & (d <= np.float32(depth_max))).sum())        # bounds the vertex count
    verts = np.zeros(cap, dtype=PLY_VERTEX)
    src = np.zeros((cap, 2), dtype=np.int32)
    cam_arr = (type(cams[0]) * n)(*cams)
    fp = C.POINTER(C.c_float)
    lib.gpo_fuse_rule.restype = C.c_longlong
    lib.gpo_fuse_rule.argtypes = [C.c_int, C.c_int, C.c_int, fp, fp, C.c_int, C.c_void_p, C.c_float, C.c_float, C.c_float,
                                  C.c_float, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_longlong, C.c_int]
    cnt = lib.gpo_fuse_rule(n, W, H, n4.ctypes.data_as(fp), None if img is None else img.ctypes.data_as(fp), ch, cam_arr,
                            depth_min, depth_max, disp_thresh, normal_thresh, num_consistent, RULES[rule], reproj_px, depth_rel,
                            r0, r1, u.ctypes.data, verts.ctypes.data, src.ctypes.data, cap, max(1, int(threads)))
    assert cnt <= cap
    return verts[:cnt], src[:cnt], u

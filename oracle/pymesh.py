"""ctypes binding of oracle/libmesh_oracle.so — the scalar C restatement of the meshing (mesh_oracle.c; DESIGN.md §24).

TEST INFRASTRUCTURE: only tests/, __graft_entry__ and tools/ may import this.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "libmesh_oracle.so")


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "mesh_oracle.c")
    hdr = os.path.join(os.path.dirname(_HERE), "include", "gipuma_b200.h")
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in (src, hdr)):
        base = ["gcc", "-O2", "-fPIC", "-shared", "-fno-fast-math", "-ffp-contract=off", "-o", LIB, src, "-lm"]
        # OpenMP over the z-slices of the integration where the toolchain has libgomp; scalar otherwise
        if subprocess.call(base[:2] + ["-fopenmp"] + base[2:], stderr=subprocess.DEVNULL) != 0:
            subprocess.check_call(base)
    return LIB


def _lib():
    lib = C.CDLL(build())
    vp = C.c_void_p
    lib.gpo_tsdf.restype = None
    lib.gpo_tsdf.argtypes = [C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_float, vp, C.c_float, C.c_float, C.c_float, C.c_int,
                             C.c_int, vp, vp, C.c_int]
    lib.gpo_mesh_extract.restype = C.c_int
    lib.gpo_mesh_extract.argtypes = [vp, vp, vp, vp, C.c_float, C.c_int, vp, C.c_int64, vp, C.c_int64,
                                     C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    return lib


def tsdf(depth, cams, origin, voxel, dims, trunc, depth_min, depth_max, slices=None, threads: int = 1):
    """gpm_tsdf_integrate restated: depth [N, H, W] float32, cams the N gpm_fuse_camera of api.fuse_cameras, dims (nx, ny,
    nz).  slices: (k0, k1), the z-slices to compute (all by default).  Returns (D [k1-k0, ny, nx] float32, Wt uint16)."""
    lib = _lib()
    dep = np.ascontiguousarray(depth, dtype=np.float32)
    n, H, W = dep.shape
    nx, ny, nz = (int(x) for x in dims)
    k0, k1 = (0, nz) if slices is None else (int(slices[0]), int(slices[1]))
    D = np.empty((k1 - k0, ny, nx), np.float32)
    Wt = np.empty((k1 - k0, ny, nx), np.uint16)
    o = np.asarray(origin, dtype=np.float32)
    d = np.asarray([nx, ny, nz], dtype=np.int32)
    cam_arr = (type(cams[0]) * n)(*cams)
    lib.gpo_tsdf(n, W, H, dep.ctypes.data, C.addressof(cam_arr), o.ctypes.data, voxel, d.ctypes.data, trunc, depth_min,
                 depth_max, k0, k1, D.ctypes.data, Wt.ctypes.data, max(1, int(threads)))
    return D, Wt


def extract(D, Wt, origin, voxel, min_weight):
    """gpm_mesh_extract restated: D float32 and Wt uint16 volumes [nz, ny, nx].  Returns (vertices [V, 3] float32,
    faces [F, 3] int32)."""
    lib = _lib()
    D = np.ascontiguousarray(D, dtype=np.float32)
    Wt = np.ascontiguousarray(Wt, dtype=np.uint16)
    nz, ny, nx = D.shape
    d = np.asarray([nx, ny, nz], dtype=np.int32)
    o = np.asarray(origin, dtype=np.float32)
    nv, nf = C.c_int64(), C.c_int64()
    for _ in range(2):                                         # count, then fill
        verts = np.zeros((max(nv.value, 1), 3), np.float32)
        faces = np.zeros((max(nf.value, 1), 3), np.int32)
        cap_v, cap_f = nv.value, nf.value
        if lib.gpo_mesh_extract(D.ctypes.data, Wt.ctypes.data, d.ctypes.data, o.ctypes.data, voxel, int(min_weight),
                                verts.ctypes.data, cap_v, faces.ctypes.data, cap_f, C.byref(nv), C.byref(nf)) != 0:
            raise MemoryError("gpo_mesh_extract")
        if nv.value <= cap_v and nf.value <= cap_f:
            break
    return verts[:nv.value], faces[:nf.value]

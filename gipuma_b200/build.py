"""Build the CUDA extension(s) in-tree for sm_90a (H100):  python -m gipuma_b200.build

  gipuma_b200/libgipuma_b200.so   the product: kernels + C-ABI (include/gipuma_b200.h)
  oracle/_ref/libhx_dropin.so     (only where the reference sources exist) the OpenCV-free stand-in for main.cpp linked
                                  against the runcuda() adapter — proves the drop-in boundary; test infrastructure.
nvcc cross-compiles without a GPU.  The .so files are git-ignored build products.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
# --use_fast_math: same arithmetic mode as the reference's build (CMakeLists.txt:23); the kernels pin every
# operation with explicit .rn.ftz intrinsics on top of it (gpm_device.cuh).
COMMON = ["-O3", "--use_fast_math", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-shared"] + ARCH
# The fusion (gpm_fuse.cu), the cloud distances (gpm_cloud.cu), the pyramid / plane upsampling (gpm_scale.cu) and the
# meshing (gpm_mesh.cu) are compiled on their own in IEEE mode: denormals kept, no contraction, so that the fusion's
# decisions are exactly those of the scalar restatement oracle/fusion_oracle.c (DESIGN.md §12), every distance is exactly
# that of the brute-force restatement oracle/pycloud.py (§13), every pyramid and upsampled value that of oracle/pyscale.py
# (§19) and every volume, vertex and face that of oracle/mesh_oracle.c (§24).
FUSE = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-ftz=false", "-prec-div=true", "-prec-sqrt=true",
        "-fmad=false", "-c"] + ARCH


def _sig(paths, extra=""):
    h = hashlib.sha1(extra.encode())
    for p in paths:
        with open(p, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def _run(cmd):
    print("[build]", " ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)


def build_library(force: bool = False) -> str:
    csrc = lambda *names: [os.path.join(HERE, "csrc", f) for f in names]
    fast = csrc("gpm_api.cu", "gpm_host.cpp", "gpm_batch.cpp", "gpm_prior.cpp")
    ieee = csrc("gpm_fuse.cu", "gpm_cloud.cu", "gpm_scale.cu", "gpm_mesh.cu")
    headers = csrc("gpm_kernels.cuh", "gpm_device.cuh", "gpm_scale.cuh") + [os.path.join(ROOT, "include", "gipuma_b200.h")]
    out = os.path.join(HERE, "libgipuma_b200.so")
    stamp = out + ".sig"
    sig = _sig(fast + ieee + headers, " ".join(COMMON + FUSE))
    if not force and os.path.exists(out) and os.path.exists(stamp) and open(stamp).read() == sig:
        return out
    with tempfile.TemporaryDirectory() as tmp:
        ieee_objs = [os.path.join(tmp, os.path.basename(s)[:-3] + ".o") for s in ieee]
        for s, o in zip(ieee, ieee_objs):
            _run([NVCC] + FUSE + ["-o", o, s])
        _run([NVCC] + COMMON + ["-o", out] + fast + ieee_objs + ["-lpthread"])
    with open(stamp, "w") as fh:
        fh.write(sig)
    return out


def build_dropin(force: bool = False):
    """Harness + runcuda adapter against the reference's own boundary headers (needs /root/reference)."""
    ref = os.environ.get("GIPUMA_REFERENCE", "/root/reference")
    if not os.path.exists(os.path.join(ref, "globalstate.h")):
        return None
    outdir = os.path.join(ROOT, "oracle", "_ref")
    os.makedirs(outdir, exist_ok=True)
    harness = os.path.join(ROOT, "oracle", "harness")
    src = [os.path.join(harness, "hx_harness.cu"), os.path.join(HERE, "csrc", "runcuda_adapter.cu"),
           os.path.join(harness, "hx_api.h"), os.path.join(ROOT, "include", "gipuma_b200.h")]
    out = os.path.join(outdir, "libhx_dropin.so")
    stamp = out + ".sig"
    sig = _sig(src, " ".join(COMMON))
    if not force and os.path.exists(out) and os.path.exists(stamp) and open(stamp).read() == sig:
        return out
    lib = build_library()
    _run([NVCC, "-O3", "-std=c++14", "-lineinfo", "-Xcompiler", "-fPIC", "-shared", "-w"] + ARCH +
         ["-I" + os.path.join(harness, "shim"), "-I" + ref, "-I" + harness, "-I" + os.path.join(ROOT, "include"),
          "-o", out, src[0], src[1], "-L" + HERE, "-lgipuma_b200", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../gipuma_b200"])
    with open(stamp, "w") as fh:
        fh.write(sig)
    return out


def build_examples(force: bool = False):
    """examples/shard_host: the C++ multi-GPU host over the C-ABI (plain g++, no CUDA headers)."""
    src = os.path.join(ROOT, "examples", "shard_host.cpp")
    out = os.path.join(ROOT, "examples", "shard_host")
    lib = build_library()
    if not force and os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(src), os.path.getmtime(lib)):
        return out
    _run(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), src, "-L" + HERE, "-lgipuma_b200", "-lpthread",
          "-Wl,-rpath,$ORIGIN/../gipuma_b200", "-o", out])
    return out


def build_all(force: bool = False):
    outs = [build_library(force), build_examples(force)]
    d = build_dropin(force)
    if d:
        outs.append(d)
    return outs


if __name__ == "__main__":
    for o in build_all(force="--force" in sys.argv):
        print(o)

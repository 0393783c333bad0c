"""Build libumr_b200.so (hand-written sm_90a kernels behind the C ABI of include/umr_b200.h).

nvcc only -- no torch / pybind headers -- so the whole library builds in seconds and
cross-compiles without a GPU.  The .so is built in-tree (umr_b200/libumr_b200.so) so the package
imports from the repository tree; it is git-ignored.

    python -m umr_b200.build [--force] [--verbose]
"""
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libumr_b200.so")
OBJ = os.path.join(PKG, "csrc", "_obj")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include"),
          "-I", CSRC]
# raster.cu must not contract a*b+c into FMA: its per-(pixel,face) arithmetic is an exact IEEE twin
# of the reference (DESIGN.md §4).  The loss kernels have no such constraint.
PER_FILE = {"raster.cu": ["-fmad=false"], "raster_f64.cu": ["-fmad=false"], "vertex.cu": ["-fmad=false"], "mesh_ops.cu": ["-fmad=false"],
            "nmr.cu": ["-fmad=false"], "voxel.cu": ["-fmad=false"]}


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    nvcc = os.environ.get("NVCC", "nvcc")
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(ROOT, "include", "umr_b200.h"))
    objs = []
    for src in sources():
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src[:-3] + ".o")
        objs.append(o)
        if force or _stale(o, [s] + headers):
            cmd = [nvcc, *ARCH, *COMMON, *PER_FILE.get(src, []), "-c", s, "-o", o]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
                print(" ".join(cmd))
            subprocess.check_call(cmd)
    if force or _stale(LIB, objs):
        cmd = [nvcc, *ARCH, "-shared", "-cudart", "static", "-o", LIB, *objs]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build("--force" in sys.argv, "--verbose" in sys.argv))

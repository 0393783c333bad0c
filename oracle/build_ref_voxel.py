"""Build the REFERENCE's own `voxelization` CUDA extension for sm_90a, as nvcc builds it (FMA contraction) and with
-fmad=false, into oracle/_ref/ -- the GPU oracle of tests/test_voxel_gpu.py and the baseline of tools/voxel_bench.py.

Same recipe and rules as build_ref_gpu.py: the two source files are read from the reference checkout, the documented
API-drift shims are applied IN A TEMP DIR (`-DAT_CHECK=TORCH_CHECK`; `faces.type()` -> `faces.scalar_type()` in the four
AT_DISPATCH_FLOATING_TYPES, `x.type().is_cuda()` -> `x.is_cuda()` in CHECK_CUDA; `.data<T>()` -> `.data_ptr<T>()`), and
only the built modules land in oracle/_ref/ (git-ignored).  Cross-compiles without a GPU; where the reference checkout is
absent, modules already built are left in place.

    python oracle/build_ref_voxel.py [--no-fma]
"""
import hashlib
import json
import os
import shutil
import subprocess
import sys
import sysconfig
import tempfile
from concurrent.futures import ThreadPoolExecutor

from build_ref_gpu import OUT, REF, _patched


def build(no_fma=False):
    """Builds (or keeps) one module; it is rebuilt when the sources, the flags, nvcc or torch change."""
    if not os.path.isdir(REF):
        return None
    import torch
    from torch.utils import cpp_extension
    name = "voxelization_ref_nofma" if no_fma else "voxelization_ref"
    os.makedirs(OUT, exist_ok=True)
    target = os.path.join(OUT, name + ".so")
    nvcc = os.environ.get("NVCC", "nvcc")
    inc = cpp_extension.include_paths(device_type="cuda") if "device_type" in cpp_extension.include_paths.__code__.co_varnames \
        else cpp_extension.include_paths(cuda=True)
    inc.append(sysconfig.get_paths()["include"])
    incs = [x for p in inc for x in ("-I", p)]
    defs = ["-DAT_CHECK=TORCH_CHECK", "-DTORCH_EXTENSION_NAME=" + name, "-DTORCH_API_INCLUDE_EXTENSION_H",
            "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI)]
    common = ["-std=c++17", "-O3", "-Xcompiler", "-fPIC", "-w"] + defs + incs
    arch = ["-gencode", "arch=compute_90a,code=sm_90a"]
    kflags = ["-fmad=false"] if no_fma else []
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    with open(os.path.join(REF, "voxelization_cuda_kernel.cu")) as f:
        cu = _patched(f.read(), "AT_DISPATCH_FLOATING_TYPES(faces.type()", "AT_DISPATCH_FLOATING_TYPES(faces.scalar_type()")
        cu = _patched(cu, ".data<scalar_t>()", ".data_ptr<scalar_t>()")
        cu = _patched(cu, ".data<int32_t>()", ".data_ptr<int32_t>()")
    with open(os.path.join(REF, "voxelization_cuda.cpp")) as f:
        cpp = _patched(f.read(), "PYBIND11_MODULE(voxelization, m)", "PYBIND11_MODULE(%s, m)" % name)
        cpp = _patched(cpp, "x.type().is_cuda()", "x.is_cuda()")
    key = hashlib.sha256(json.dumps([nvcc, arch, common, kflags, libdir, torch.__version__, cu, cpp]).encode()).hexdigest()
    stamp = target + ".key"
    if os.path.exists(target) and os.path.exists(stamp):
        with open(stamp) as f:
            if f.read().strip() == key:
                return target
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, "k.cu"), "w") as f:
            f.write(cu)
        with open(os.path.join(tmp, "b.cpp"), "w") as f:
            f.write(cpp)
        subprocess.check_call([nvcc, *arch, *common, *kflags, "-c", os.path.join(tmp, "k.cu"), "-o", os.path.join(tmp, "k.o")])
        subprocess.check_call([nvcc, *arch, *common, "-x", "cu", "-c", os.path.join(tmp, "b.cpp"), "-o",
                               os.path.join(tmp, "b.o")])
        so = os.path.join(tmp, name + ".so")
        subprocess.check_call([nvcc, *arch, "-shared", "-o", so, os.path.join(tmp, "k.o"), os.path.join(tmp, "b.o"),
                               "-L", libdir, "-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda",
                               "-Xlinker", "-rpath", "-Xlinker", libdir])
        if os.path.exists(stamp):
            os.remove(stamp)
        shutil.move(so, target)
    with open(stamp, "w") as f:
        f.write(key + "\n")
    return target


def build_all():
    """Both modules (FMA-contracted and -fmad=false), compiled concurrently."""
    with ThreadPoolExecutor(2) as ex:
        return list(ex.map(build, (False, True)))


if __name__ == "__main__":
    print(build("--no-fma" in sys.argv))

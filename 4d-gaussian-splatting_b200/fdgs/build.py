"""In-tree build of the native pieces (explicit nvcc / g++ command lines, no JIT cache).

  libfdgs.so   the product: CUDA kernels + C-ABI (include/fdgs.h), sm_90a only
  fdgs_C.so    thin torch extension over the C-ABI (the three entry points of the reference's
               `_C`, reference: diff-gaussian-rasterization/ext.cpp:15-19, their extended pair
               rasterize_gaussians_ext / _backward_ext, and the training-step bindings)

Both land in `4d-gaussian-splatting_b200/fdgs/lib/` (git-ignored).  Nothing here falls back to a CPU or PyTorch implementation: if the libraries are
missing, importing `fdgs` raises.
"""
import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REPO_DIR = os.path.dirname(PKG_DIR)
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_DIR = os.path.join(PKG_DIR, "fdgs", "lib")
OBJ_DIR = os.path.join(LIB_DIR, "obj")

CU_SOURCES = ["preprocess_fwd.cu", "binning.cu", "blend_fwd.cu", "blend_bwd.cu", "preprocess_bwd.cu", "exchange.cu", "loss.cu", "optim.cu", "knn.cu", "sky.cu", "densify.cu", "regularize.cu", "metrics.cu", "fdgs_api.cu"]
HEADERS = ["fdgs_common.cuh", "fdgs_internal.h", "ssim_common.cuh", os.path.join(REPO_DIR, "include", "fdgs.h")]

NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]
# the flags the objects in lib/ were compiled with: objects built with other flags (another target architecture) are
# rebuilt even when they are newer than their sources
FLAGS_STAMP = os.path.join(LIB_DIR, "nvcc_flags.txt")


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def _run(cmd, verbose):
    if verbose:
        print("[fdgs build]", " ".join(cmd), flush=True)
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("command failed (%d): %s\n%s" % (r.returncode, " ".join(cmd), r.stdout))
    return r.stdout


def build_lib(force=False, verbose=True):
    """nvcc -> libfdgs.so (every .cu compiled for sm_90a with -lineinfo)."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    stamp = " ".join(NVCC_FLAGS)
    if not os.path.exists(FLAGS_STAMP) or open(FLAGS_STAMP).read() != stamp:
        force = True
    hdrs = [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    jobs = []
    objs = []
    for s in CU_SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ_DIR, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _newer(obj, [src] + hdrs):
            jobs.append([_nvcc()] + NVCC_FLAGS + ["-c", src, "-o", obj])
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(lambda c: _run(c, verbose), jobs))
    lib = os.path.join(LIB_DIR, "libfdgs.so")
    if force or jobs or not os.path.exists(lib):
        _run([_nvcc(), "-shared", "-o", lib] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"], verbose)
        with open(FLAGS_STAMP, "w") as f:
            f.write(stamp)
    return lib


def build_ext(force=False, verbose=True):
    """g++ -> fdgs_C.so (pybind11 module linking libfdgs.so and libtorch)."""
    import torch
    from torch.utils import cpp_extension as ce

    lib = build_lib(force=force, verbose=verbose)
    src = os.path.join(CSRC, "torch_ext.cpp")
    out = os.path.join(LIB_DIR, "fdgs_C.so")
    if not (force or _newer(out, [src, lib, os.path.join(REPO_DIR, "include", "fdgs.h")])):
        return out
    cuda_home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    inc = ce.include_paths() + [sysconfig.get_paths()["include"], os.path.join(cuda_home, "include")]
    torch_lib = os.path.join(os.path.dirname(torch.__file__), "lib")
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-DTORCH_EXTENSION_NAME=fdgs_C",
           "-DTORCH_API_INCLUDE_EXTENSION_H", "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI),
           "-Wno-deprecated-declarations"]
    for i in inc:
        cmd += ["-isystem", i]
    cmd += [src, "-o", out, "-L" + LIB_DIR, "-lfdgs", "-L" + torch_lib, "-lc10", "-lc10_cuda", "-ltorch_cpu",
            "-ltorch_cuda", "-ltorch", "-ltorch_python", "-L" + os.path.join(cuda_home, "lib64"), "-lcudart",
            "-Wl,-rpath,$ORIGIN", "-Wl,-rpath," + torch_lib]
    _run(cmd, verbose)
    return out


def build_all(force=False, verbose=True):
    build_lib(force=force, verbose=verbose)
    build_ext(force=force, verbose=verbose)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv)

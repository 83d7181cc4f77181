"""Build libsassd_b200.so (all CUDA kernels + the C ABI) in-tree with nvcc for sm_90a (H100).

    python -m sassd_b200.build [--force]

nvcc cross-compiles without a GPU; the shared object and the object files under
build/ are build products (git-ignored)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsassd_b200.so")
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC", "-diag-suppress", "550"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps():
    d = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    d.append(os.path.join(os.path.dirname(HERE), "include", "sassd_b200.h"))
    return d


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(s) > t for s in _deps())


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)

    def cc(src):
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        hdr_t = max(os.path.getmtime(p) for p in _deps() if not p.endswith(".cu"))
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_t):
            cmd = ["nvcc"] + NVCC_FLAGS + ["-c", src, "-o", obj]
            if verbose:
                print(" ".join(cmd))
            subprocess.check_call(cmd)
        return obj
    with ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(cc, sources()))
    cmd = ["nvcc", "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))

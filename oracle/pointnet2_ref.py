"""ORACLE build recipe for the reference's pointnet2 interpolation kernels — test infrastructure only.

``build()``: when a checkout of the original SA-SSD project is present (SASSD_REFERENCE_ROOT, default
/root/reference, as for oracle/build.py), compile its mmdet/ops/pointnet2/src/interpolate_gpu.cu *where it lies*,
unmodified, for sm_90a into oracle/_ref/libpointnet2_ref.so (git-ignored).  The file's
``<torch/serialize/tensor.h>`` include resolves against torch's headers; nothing of torch is linked.  The library
exports the C++-mangled ``three_nn_kernel_launcher_fast`` / ``three_interpolate_kernel_launcher_fast``, which
tests/test_point_aux.py calls through ctypes to check sassd_three_nn bit for bit.  No reference source is copied.
"""
import os
import subprocess

from .build import HERE, REF_ROOT_DEFAULT, _newer

SRC_REL = os.path.join("mmdet", "ops", "pointnet2", "src", "interpolate_gpu.cu")


def path():
    return os.path.join(HERE, "_ref", "libpointnet2_ref.so")


def build(force=False):
    """Returns the library's path, or None if it can neither be built (no checkout of the original project) nor
    found prebuilt."""
    out = path()
    root = os.environ.get("SASSD_REFERENCE_ROOT") or REF_ROOT_DEFAULT
    src = os.path.join(root, SRC_REL)
    if os.path.isfile(src) and (force or _newer(out, [src])):
        from torch.utils.cpp_extension import include_paths
        os.makedirs(os.path.dirname(out), exist_ok=True)
        cmd = ["nvcc", "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-shared",
               "-Xcompiler", "-fPIC", "-o", out, src]
        for p in include_paths():
            cmd += ["-I", p]
        subprocess.check_call(cmd)
    return out if os.path.isfile(out) else None


if __name__ == "__main__":
    print(build(force=True))

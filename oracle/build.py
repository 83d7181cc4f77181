"""ORACLE build recipe — test infrastructure only.

* ``build_oracle()``: gcc -> oracle/liboracle.so (voxelize.c + nms.c, fp contraction
  off, no fast-math).
* ``build_ref()``: when a checkout of the original SA-SSD project is present
  (SASSD_REFERENCE_ROOT, default /root/reference), compile its rotated-NMS CUDA source
  *where it lies* (mmdet/ops/iou3d/src/iou3d_kernel.cu, unmodified, sm_90a) into
  oracle/_ref/libiou3d_ref.so (git-ignored).  No reference source is copied into
  the repo.  bench.py --impl reference-gpu uses the library; tests/golden/make_golden_nms.py
  ran it once and the suppression masks it computed are committed as
  tests/golden/nms_ref.npz, so the tests do not need it.
  The other reference native code on this path (spconv v1.0) is third-party and
  absent; the numba voxelizer's outputs are committed as tests/golden/*.npz.
"""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
REF_REL = os.path.join("mmdet", "ops", "iou3d", "src", "iou3d_kernel.cu")


REF_ROOT_DEFAULT = "/root/reference"     # where the original project is checked out beside this one


def ref_src():
    root = os.environ.get("SASSD_REFERENCE_ROOT") or REF_ROOT_DEFAULT
    return os.path.join(root, REF_REL)


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def build_oracle(force=False):
    out = os.path.join(HERE, "liboracle.so")
    srcs = [os.path.join(HERE, "voxelize.c"), os.path.join(HERE, "nms.c")]
    if force or _newer(out, srcs):
        cmd = ["gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off", "-fno-fast-math",
               "-o", out] + srcs + ["-lm"]
        subprocess.check_call(cmd)
    return out


def ref_path():
    return os.path.join(HERE, "_ref", "libiou3d_ref.so")


def build_ref(force=False):
    """Returns the path of the reference NMS library, or None if it can neither be
    built (no checkout of the original project) nor found prebuilt."""
    out = ref_path()
    src = ref_src()
    if src and os.path.isfile(src) and (force or _newer(out, [src])):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        cmd = ["nvcc", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-shared",
               "-Xcompiler", "-fPIC", "-o", out, src]
        subprocess.check_call(cmd)
    return out if os.path.isfile(out) else None


if __name__ == "__main__":
    print(build_oracle(force=True))
    print(build_ref(force=True))

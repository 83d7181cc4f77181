"""ORACLE build recipe for the reference's ``pts_in_boxes3d`` — test infrastructure only.

``build()``: when a checkout of the original SA-SSD project is present (SASSD_REFERENCE_ROOT, default /root/reference,
as for oracle/build.py), compile its mmdet/ops/points_op/src/points_op.cpp *where it lies*, unmodified, as a CPU torch
extension into oracle/_ref/ (git-ignored).  The file spells its check macro AT_CHECK, which current torch no longer
defines, so the command line maps it to TORCH_CHECK.  x86-64 g++ without -march emits no FMA, as the reference's own
build.  ``load()`` imports the extension; its ``pts_in_boxes3d(pts [N,3], boxes [M,7], flags [M,N] int32, reg [N,3])``
is the oracle of sassd_points_in_boxes.  No reference source is copied.
"""
import glob
import importlib.util
import os

from .build import HERE, REF_ROOT_DEFAULT, _newer

SRC_REL = os.path.join("mmdet", "ops", "points_op", "src", "points_op.cpp")
NAME = "points_op_ref"


def out_dir():
    return os.path.join(HERE, "_ref", "points_op")


def path():
    found = glob.glob(os.path.join(out_dir(), NAME + "*.so"))
    return found[0] if found else None


def build(force=False):
    """Returns the extension's path, or None if it can neither be built (no checkout of the original project) nor
    found prebuilt."""
    root = os.environ.get("SASSD_REFERENCE_ROOT") or REF_ROOT_DEFAULT
    src = os.path.join(root, SRC_REL)
    out = path()
    if os.path.isfile(src) and (force or out is None or _newer(out, [src])):
        from torch.utils.cpp_extension import load as load_ext
        os.makedirs(out_dir(), exist_ok=True)
        load_ext(NAME, [src], extra_cflags=["-O2", "-DAT_CHECK=TORCH_CHECK"], build_directory=out_dir(), verbose=False)
        out = path()
    return out


def load():
    """The built extension module, or None."""
    p = path()
    if p is None:
        return None
    import torch  # noqa: F401  (the extension links against torch's libraries)
    spec = importlib.util.spec_from_file_location(NAME, p)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build(force=True))

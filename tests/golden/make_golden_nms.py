"""Generate tests/golden/nms_ref.npz: the suppression bitmasks that the ORIGINAL project's rotated-NMS CUDA kernel
(mmdet/ops/iou3d/src/iou3d_kernel.cu, nmsLauncher, unmodified) computes for the box sets of
tests/test_gpu_parity.py::test_nms_mask_and_keep, together with those (sorted BEV) inputs.  The test compares the
product's kernel with these masks bit for bit.  Needs a CUDA device and the reference library built by
oracle/build.py:build_ref():

    python -m oracle.build          # SASSD_REFERENCE_ROOT = the original project, default /root/reference
    python tests/golden/make_golden_nms.py [out.npz]
"""
import ctypes
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build as ob  # noqa: E402
from tests.test_gpu_parity import NMS_CASES, NMS_THR, _sorted_bev  # noqa: E402


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "nms_ref.npz")
    path = ob.build_ref()
    assert path, "reference NMS library not built (no checkout of the original project; see oracle/build.py)"
    fn = getattr(ctypes.CDLL(path), "_Z11nmsLauncherPKfPyif")
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_float]
    fn.restype = None
    dev = torch.device("cuda:0")
    arrays = {}
    for n, seed in NMS_CASES:
        bev = _sorted_bev(n, seed)
        d_bev = bev.to(dev)
        rmask = torch.zeros((n, (n + 63) // 64), dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        fn(ctypes.c_void_p(d_bev.data_ptr()), ctypes.c_void_p(rmask.data_ptr()), n, ctypes.c_float(NMS_THR))
        torch.cuda.synchronize()
        arrays["bev_%d_%d" % (n, seed)] = bev.numpy()
        arrays["mask_%d_%d" % (n, seed)] = rmask.cpu().numpy().view(np.uint64)
    np.savez_compressed(out, **arrays)
    print("wrote", out)


if __name__ == "__main__":
    main()

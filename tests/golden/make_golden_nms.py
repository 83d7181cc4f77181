"""Generate tests/golden/nms_ref.npz: the suppression bitmasks that the ORIGINAL project's rotated-NMS CUDA kernel
(mmdet/ops/iou3d/src/iou3d_kernel.cu, nmsLauncher, unmodified) computes for the box sets of
tests/test_gpu_parity.py::test_nms_mask_and_keep and of the clustered scenes at the NMS capacity of
tests/test_detection_tail.py (n = 2048, 4095, 4096; IoU thresholds 0.1 and 0.0), together with those (sorted BEV)
inputs - for the large scenes their sha256 and only the masks' upper triangle, lzma-compressed.  The tests compare
the product's kernel with these masks bit for bit.  Needs a CUDA device and the reference library built by
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
from tests.test_detection_tail import (TAIL_NMS_CASES, TAIL_NMS_THRS, bev_digest, pack_reference_mask,  # noqa: E402
                                       tail_nms_inputs)
from tests.test_gpu_parity import NMS_CASES, NMS_THR, _sorted_bev  # noqa: E402


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "nms_ref.npz")
    path = ob.build_ref()
    assert path, "reference NMS library not built (no checkout of the original project; see oracle/build.py)"
    fn = getattr(ctypes.CDLL(path), "_Z11nmsLauncherPKfPyif")
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_float]
    fn.restype = None
    dev = torch.device("cuda:0")

    def ref_mask(bev, thr):
        n = bev.shape[0]
        d_bev = bev.to(dev)
        rmask = torch.zeros((n, (n + 63) // 64), dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        fn(ctypes.c_void_p(d_bev.data_ptr()), ctypes.c_void_p(rmask.data_ptr()), n, ctypes.c_float(thr))
        torch.cuda.synchronize()
        return rmask.cpu().numpy().view(np.uint64)

    arrays = {}
    for n, seed in NMS_CASES:
        bev = _sorted_bev(n, seed)
        arrays["bev_%d_%d" % (n, seed)] = bev.numpy()
        arrays["mask_%d_%d" % (n, seed)] = ref_mask(bev, NMS_THR)
    for n in TAIL_NMS_CASES:
        bev = tail_nms_inputs(n)[3]
        # the large cases keep the file small: their inputs by digest (the test rebuilds the scene), their masks'
        # upper triangle lzma-compressed
        arrays["tail_bev_sha256_%d" % n] = np.array(bev_digest(bev))
        for thr in TAIL_NMS_THRS:
            arrays["tail_mask_%d_%g" % (n, thr)] = pack_reference_mask(ref_mask(torch.from_numpy(bev), thr))
    np.savez_compressed(out, **arrays)
    print("wrote", out)


if __name__ == "__main__":
    main()

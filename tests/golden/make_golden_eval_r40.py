"""Generate tests/golden/eval_r40.npz: the REFERENCE's eval_class_v3 precision and orientation arrays
(mmdet/core/evaluation/kitti_eval.py:549-657) on the annotations of tests/golden/eval.npz, for the three metrics, so
that AP at 40 recall positions can be checked against the reference's own 41 precision samples.  The rotated-IoU
kernel is numba.cuda code; without a GPU it runs in numba's CUDA simulator:

    NUMBA_ENABLE_CUDASIM=1 python tests/golden/make_golden_eval_r40.py

Keys: ``prec_<metric>`` [class, difficulty, min_overlap, 41] for metric 0 (bbox), 1 (bev), 2 (3d) and ``orient_0``
(AOS samples of the bbox metric), for classes (0, 1, 2) and both official overlap sets.
"""
import importlib.util
import os
import sys

import numpy as np
import numpy.ma  # noqa: F401  (before make_golden's np.bool shim)
import numba  # noqa: F401

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import import_reference_mmdet  # noqa: E402

KEYS = ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location', 'rotation_y')


def main():
    assert os.environ.get("NUMBA_ENABLE_CUDASIM") == "1", "run with NUMBA_ENABLE_CUDASIM=1 (no GPU here)"
    import_reference_mmdet()
    for k in list(sys.modules):
        if k.startswith("mmdet.core.post_processing"):
            del sys.modules[k]
    spec = importlib.util.spec_from_file_location(
        "mmdet.core.post_processing.rotate_nms_gpu", "/root/reference/mmdet/core/post_processing/rotate_nms_gpu.py")
    m = importlib.util.module_from_spec(spec); sys.modules[spec.name] = m; spec.loader.exec_module(m)
    spec = importlib.util.spec_from_file_location("ref_kitti_eval", "/root/reference/mmdet/core/evaluation/kitti_eval.py")
    ke = importlib.util.module_from_spec(spec); spec.loader.exec_module(ke)

    g = np.load(os.path.join(HERE, "eval.npz"))
    n = int(g["nframes"])
    gts = [{k: g["gt%d_%s" % (i, k)] for k in KEYS} for i in range(n)]
    dts = [{k: g["dt%d_%s" % (i, k)] for k in KEYS + ("score",)} for i in range(n)]
    classes = [0, 1, 2]
    overlap = np.stack([np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7, 0.7, 0.7]] * 3),
                        np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5],
                                  [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5]])], 0)[:, :, classes]
    out = {}
    for metric in (0, 1, 2):
        ret = ke.eval_class_v3(gts, dts, classes, [0, 1, 2], metric, overlap, metric == 0)
        out["prec_%d" % metric] = np.asarray(ret["precision"])
        if metric == 0:
            out["orient_0"] = np.asarray(ret["orientation"])
    np.savez_compressed(os.path.join(HERE, "eval_r40.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()

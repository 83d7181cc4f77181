"""Generate tests/golden/eval_coco.npz: the REFERENCE's COCO-style KITTI evaluation (get_coco_eval_result and
do_coco_style_eval, mmdet/core/evaluation/kitti_eval.py:711-729, :853-930) on the annotations of
tests/golden/eval.npz.  The rotated-IoU kernel is numba.cuda code; without a GPU it runs in numba's CUDA simulator:

    NUMBA_ENABLE_CUDASIM=1 python tests/golden/make_golden_eval_coco.py

The reference passes np.linspace a float ``num`` (its class_to_range rows are float arrays), which NumPy >= 1.18
rejects; the one shim here makes that call take int(num).  Nothing else is changed.

Keys, for each class list tag (``c012``: classes 0, 1, 2; ``car``: class 0 alone): ``text_<tag>`` (the printed table)
and ``bbox_<tag>``, ``bev_<tag>``, ``d3_<tag>``, ``aos_<tag>`` ([class, difficulty], do_coco_style_eval's arrays).
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

    linspace = np.linspace

    def linspace_int_num(start, stop, num=50, *a, **k):
        return linspace(start, stop, int(num), *a, **k)
    np.linspace = linspace_int_num          # the shim: numba-compiled code never calls linspace

    g = np.load(os.path.join(HERE, "eval.npz"))
    n = int(g["nframes"])
    gts = [{k: g["gt%d_%s" % (i, k)] for k in KEYS} for i in range(n)]
    dts = [{k: g["dt%d_%s" % (i, k)] for k in KEYS + ("score",)} for i in range(n)]
    out = {}
    for tag, classes in (("c012", [0, 1, 2]), ("car", [0])):
        out["text_" + tag] = np.array(ke.get_coco_eval_result(gts, dts, classes))
        ranges = np.zeros([3, 3, len(classes)])
        for i, c in enumerate(classes):
            ranges[:, :, i] = np.array({0: [0.5, 0.95, 10], 1: [0.25, 0.7, 10], 2: [0.25, 0.7, 10]}[c])[:, None]
        bbox, bev, d3, aos = ke.do_coco_style_eval(gts, dts, classes, ranges, True)
        out.update({"bbox_" + tag: bbox, "bev_" + tag: bev, "d3_" + tag: d3, "aos_" + tag: aos})
    np.linspace = linspace
    np.savez_compressed(os.path.join(HERE, "eval_coco.npz"), **out)
    print({k: v.shape for k, v in out.items()})
    print(str(out["text_c012"]))


if __name__ == "__main__":
    main()

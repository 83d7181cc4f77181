"""Generate tests/golden/eval_bootstrap.npz: the REFERENCE's KITTI evaluation (mmdet/core/evaluation/kitti_eval.py) on
bootstrap replicates of the frames of tests/golden/eval_ranges.npz (eval.npz's frames and the range fixture's).  The
rotated-IoU kernel is numba.cuda code; without a GPU it runs in numba's CUDA simulator:

    NUMBA_ENABLE_CUDASIM=1 python tests/golden/make_golden_eval_bootstrap.py

A replicate is a list of frames drawn with replacement; the unmodified reference evaluates the GT and detection lists of
it: eval_class_v3 + get_mAP_v2 at the official overlaps (do_eval_v2) and do_coco_style_eval, compute_aos decided as
get_official_eval_result decides it (from the list's first frame with detections).

Keys: ``idx`` [R, F] the replicates' frame indices: 8 rows of np.random.RandomState(7).randint(0, F, F), then the
identity, one frame repeated F times, and a draw from the frames without a Pedestrian GT; ``aos`` [R] compute_aos; per
replicate r ``r<r>_<bbox|bev|d3|aos>`` (do_eval_v2's [class, difficulty, 2 overlap rows]; aos absent without it) and
``r<r>_coco_<...>`` (do_coco_style_eval's [class, difficulty]).
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
CLASSES = [0, 1, 2]
OVERLAP = np.stack([np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7, 0.7, 0.7]] * 3),
                    np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5],
                              [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5]])], 0)[:, :, CLASSES]
COCO = {0: [0.5, 0.95, 10], 1: [0.25, 0.7, 10], 2: [0.25, 0.7, 10]}


def replicates(gts):
    n = len(gts)
    rs = np.random.RandomState(7)
    rows = [rs.randint(0, n, n) for _ in range(8)]
    rows.append(np.arange(n))
    busy = max(range(n), key=lambda f: (np.asarray(gts[f]["name"]) == "Car").sum())
    rows.append(np.full(n, busy))
    no_ped = np.array([f for f in range(n) if not (np.asarray(gts[f]["name"]) == "Pedestrian").any()])
    rows.append(no_ped[np.random.RandomState(8).randint(0, len(no_ped), n)])
    return np.stack(rows).astype(np.int64)


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
    np.linspace = linspace_int_num          # the reference passes a float num (see make_golden_eval_coco.py)

    g = np.load(os.path.join(HERE, "eval_ranges.npz"))
    n = int(g["nframes"])
    gts = [{k: g["gt%d_%s" % (i, k)] for k in KEYS} for i in range(n)]
    dts = [{k: g["dt%d_%s" % (i, k)] for k in KEYS + ("score",)} for i in range(n)]
    idx = replicates(gts)
    ranges = np.zeros([3, 3, len(CLASSES)])
    for i, c in enumerate(CLASSES):
        ranges[:, :, i] = np.array(COCO[c])[:, None]
    out = {"idx": idx, "aos": np.zeros(len(idx), bool)}
    for r, row in enumerate(idx):
        gr, dr = [gts[f] for f in row], [dts[f] for f in row]
        compute_aos = False
        for anno in dr:                      # get_official_eval_result's decision (kitti_eval.py:818-823)
            if anno['alpha'].shape[0] != 0:
                compute_aos = bool(anno['alpha'][0] != -10)
                break
        out["aos"][r] = compute_aos
        for tag, ap in (("", ke.do_eval_v2(gr, dr, CLASSES, OVERLAP, compute_aos, [0, 1, 2])),
                        ("coco_", ke.do_coco_style_eval(gr, dr, CLASSES, ranges, compute_aos))):
            for key, v in zip(("bbox", "bev", "d3", "aos"), ap):
                if v is not None:
                    out["r%d_%s%s" % (r, tag, key)] = np.asarray(v)
        print(r, out["r%d_d3" % r][:, 1, 0])
    np.linspace = linspace
    np.savez_compressed(os.path.join(HERE, "eval_bootstrap.npz"), **out)


if __name__ == "__main__":
    main()

"""Generate tests/golden/eval_ranges.npz: the REFERENCE's KITTI evaluation (mmdet/core/evaluation/kitti_eval.py)
per range bin, on the annotations of tests/golden/eval.npz plus frames that populate every bin.  The rotated-IoU
kernel is numba.cuda code; without a GPU it runs in numba's CUDA simulator:

    NUMBA_ENABLE_CUDASIM=1 python tests/golden/make_golden_eval_ranges.py

The reference evaluator is not changed.  A bin's semantics (a GT or detection of the class outside the bin is ignored)
come from transformed annotations, class by class: ``occluded = 3`` on each out-of-bin GT of the class (harder than
every difficulty) and ``bbox[3] = bbox[1]`` on each out-of-bin detection of the class (lower than every minimum
height).  The second changes the 2-D boxes, so only the BEV and 3-D metrics are kept.

Keys: the annotations (``nframes``, ``gt<i>_<key>``, ``dt<i>_<key>``), ``edges``, and for class c, bin b and metric m
(1 BEV, 2 3-D) ``prec_c<c>_b<b>_m<m>`` (eval_class_v3's precision [1, 3 difficulties, 2 overlap rows, 41]) and
``ap_c<c>_b<b>_m<m>`` (get_mAP_v2 of it); for class c, difficulty d and metric m (0, 1, 2) ``stat_c<c>_d<d>_m<m>``:
compute_statistics_jit's (tp, fp, fn) summed over the frames over the whole range, compute_fp=True at a threshold
below every score and the class's first official min overlap.
"""
import copy
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
EDGES = (0.0, 4.0, 20.0, 40.0, np.inf)       # [0, 4) holds no GT: an empty bin
SIZES = {'Car': (3.9, 1.56, 1.6), 'Pedestrian': (0.8, 1.73, 0.6), 'Cyclist': (1.76, 1.73, 0.6)}   # l, h, w
OVERLAP = np.stack([np.array([[0.7, 0.5, 0.5]] * 3), np.array([[0.7, 0.5, 0.5], [0.5, 0.25, 0.25],
                                                              [0.5, 0.25, 0.25]])], 0)


def _rows(objs, score=False):
    """Annotation dict of (name, x, z, ry, score) objects, camera height 1.6, 2-D boxes from a pinhole f = 720."""
    n = len(objs)
    names = np.array([o[0] for o in objs], dtype=str).reshape(n)
    loc = np.array([[o[1], 1.6, o[2]] for o in objs], np.float64).reshape(n, 3)
    dims = np.array([SIZES[o[0]] for o in objs], np.float64).reshape(n, 3)
    h2d = 720.0 * dims[:, 1] / loc[:, 2]
    w2d = 720.0 * dims[:, 0] / loc[:, 2]
    cx = 620 + 720 * loc[:, 0] / loc[:, 2]
    bbox = np.stack([cx - w2d / 2, 190 - h2d / 2, cx + w2d / 2, 190 + h2d / 2], 1).reshape(n, 4)
    a = dict(name=names, truncated=np.zeros(n), occluded=np.zeros(n, np.int64),
             alpha=np.array([o[3] for o in objs], np.float64).reshape(n), bbox=bbox, dimensions=dims, location=loc,
             rotation_y=np.array([o[3] for o in objs], np.float64).reshape(n))
    if score:
        a["score"] = np.array([o[4] for o in objs], np.float64).reshape(n)
    return a


def extra_frames():
    """Frames with GT exactly at an edge (x = 12, z = 16: 20 m), detection / GT pairs straddling the 20 m and 40 m
    edges both ways, objects in every non-empty bin and a lone detection in the empty bin [0, 4)."""
    frames = [
        ([('Car', 12.0, 16.0, 0.1), ('Car', 0.0, 19.9, 0.0)],
         [('Car', 12.05, 16.02, 0.12, 0.9), ('Car', 0.0, 20.1, 0.02, 0.8), ('Car', 1.0, 2.0, 0.0, 0.7)]),
        ([('Car', 0.0, 40.05, 0.3), ('Car', -5.0, 30.0, 1.0), ('Pedestrian', 2.0, 19.95, 0.0)],
         [('Car', 0.0, 39.95, 0.31, 0.6), ('Car', -5.1, 30.1, 1.05, 0.95), ('Pedestrian', 2.0, 20.05, 0.1, 0.5)]),
        ([('Cyclist', -3.0, 12.0, 0.5), ('Cyclist', 4.0, 45.0, -0.5), ('Pedestrian', -1.0, 8.0, 2.0)],
         [('Cyclist', -3.05, 12.1, 0.45, 0.85), ('Cyclist', 4.05, 44.9, -0.4, 0.65),
          ('Pedestrian', -1.02, 8.03, 2.1, 0.75), ('Car', 6.0, 50.0, 0.0, 0.4)]),
        ([('Car', 10.0, 55.0, -1.0), ('Car', -8.0, 36.0, 2.5), ('Pedestrian', 0.5, 39.98, 0.0)],
         [('Car', 10.1, 55.2, -1.1, 0.55), ('Car', -8.05, 36.05, 2.45, 0.9), ('Pedestrian', 0.5, 40.02, 0.0, 0.6)]),
    ]
    return [_rows(g) for g, _ in frames], [_rows(d, True) for _, d in frames]


def ground_range(a):
    loc = np.asarray(a["location"], np.float64).reshape(-1, 3)
    return np.sqrt(loc[:, 0] * loc[:, 0] + loc[:, 2] * loc[:, 2])


def binned(annos, cls, lo, hi, gt):
    """The annotations with the bin's semantics for class ``cls`` in the reference's own terms."""
    out = []
    for a in annos:
        a = copy.deepcopy(a)
        r = ground_range(a)
        out_of_bin = (np.char.lower(np.asarray(a["name"], str)) == cls.lower()) & ~((lo <= r) & (r < hi))
        if gt:
            a["occluded"] = np.where(out_of_bin, 3, a["occluded"])
        else:
            a["bbox"] = a["bbox"].copy()
            a["bbox"][out_of_bin, 3] = a["bbox"][out_of_bin, 1]
        out.append(a)
    return out


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
    eg, ed = extra_frames()
    gts, dts = gts + eg, dts + ed
    out = {"nframes": np.array(len(gts)), "edges": np.array(EDGES)}
    for i, (a, b) in enumerate(zip(gts, dts)):
        out.update({"gt%d_%s" % (i, k): v for k, v in a.items()})
        out.update({"dt%d_%s" % (i, k): v for k, v in b.items()})
    names = {0: "Car", 1: "Pedestrian", 2: "Cyclist"}
    for c in (0, 1, 2):
        for b, (lo, hi) in enumerate(zip(EDGES[:-1], EDGES[1:])):
            gb, db = binned(gts, names[c], lo, hi, True), binned(dts, names[c], lo, hi, False)
            for metric in (1, 2):
                ret = ke.eval_class_v3(gb, db, [c], [0, 1, 2], metric, OVERLAP[:, :, [c]])
                out["prec_c%d_b%d_m%d" % (c, b, metric)] = ret["precision"]
                out["ap_c%d_b%d_m%d" % (c, b, metric)] = ke.get_mAP_v2(ret["precision"])
    for metric in (0, 1, 2):
        overlaps = ke.calculate_iou_partly(dts, gts, metric, 50)[0]
        for c in (0, 1, 2):
            for d in (0, 1, 2):
                gt_datas, dt_datas, ign_gt, ign_dt, dcs, _, _ = ke._prepare_data(gts, dts, c, d)
                tot = np.zeros(3, np.int64)
                for i in range(len(gts)):
                    tp, fp, fn, _, _ = ke.compute_statistics_jit(
                        overlaps[i], gt_datas[i], dt_datas[i], ign_gt[i], ign_dt[i], dcs[i], metric,
                        OVERLAP[0, metric, c], -np.inf, compute_fp=True)
                    tot += (tp, fp, fn)
                out["stat_c%d_d%d_m%d" % (c, d, metric)] = tot
    np.savez_compressed(os.path.join(HERE, "eval_ranges.npz"), **out)
    print({k: v for k, v in out.items() if k.startswith(("ap_", "stat_"))})


if __name__ == "__main__":
    main()

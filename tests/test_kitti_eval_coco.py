"""COCO-style KITTI AP (kitti_eval.coco_eval / get_coco_eval_result, the reference's get_coco_eval_result) and the
device evaluator (csrc/kitti_match.cu) that serves it and the official tables.

* CPU: the host path (the oracle's rotated overlaps injected) equals the reference's table and arrays
  (tests/golden/eval_coco.npz, make_golden_eval_coco.py); the K-set functions equal K single calls; argument errors.
* GPU: the device evaluator equals the goldens (COCO, official R11 and R40) and equals the host path bit for bit on
  sets built to stress it: empty frames, DontCare-only frames, tied scores, overlaps between a linspace value and its
  rounded decimal, a frame of more than 128 detections, K = 1, 4 and 10 sets, a single class.  The driver's --coco.
"""
import copy
import ctypes
import math
import os
import sys

import numpy as np
import pytest

from oracle import kitti_eval as O
from sassd_b200 import kitti_eval as K
from tests.test_kitti_eval import GOLD, _annos

HERE = os.path.dirname(os.path.abspath(__file__))
COCO_GOLD = os.path.join(HERE, "golden", "eval_coco.npz")
CLASS_SETS = (("c012", [0, 1, 2]), ("car", [0]))


def _gold():
    return _annos(np.load(GOLD)), np.load(COCO_GOLD)


def _same_coco(got, gold, tag):
    text, ap = got
    assert text == str(gold["text_" + tag])
    for k in ("bbox", "bev", "d3", "aos"):
        np.testing.assert_array_equal(ap[k], gold["%s_%s" % (k, tag)], err_msg=k)


def _same_tables(a, b):
    assert a.keys() == b.keys()
    for key in a:
        assert a[key][0] == b[key][0], key
        for k in ("bbox", "bev", "d3", "aos"):
            if a[key][1][k] is None or b[key][1][k] is None:
                assert a[key][1][k] is None and b[key][1][k] is None, (key, k)
            else:
                np.testing.assert_array_equal(a[key][1][k], b[key][1][k], err_msg="%s %s" % (key, k))


# ------------------------------------------------------------------------------------------------------------ CPU
def test_host_path_equals_the_reference_coco_table():
    (gts, dts), gold = _gold()
    for tag, classes in CLASS_SETS:
        _same_coco(K.coco_eval(gts, dts, classes, overlap_fn=O.rotate_iou_eval), gold, tag)
    assert K.get_coco_eval_result(gts, dts, ["Car", "Pedestrian", "Cyclist"],
                                  overlap_fn=O.rotate_iou_eval) == str(gold["text_c012"])
    assert K.get_coco_eval_result(gts, dts, "Car", overlap_fn=O.rotate_iou_eval) == str(gold["text_car"])
    assert str(gold["text_c012"]).startswith("Car coco AP@0.50:0.05:0.95:\nbbox AP:")
    assert "Pedestrian coco AP@0.25:0.05:0.70:" in str(gold["text_c012"])


def test_coco_overlaps_are_the_hosts_linspace_values():
    mo = K.coco_min_overlaps([0, 1, 2])
    assert mo.shape == (10, 3, 3)
    np.testing.assert_array_equal(mo[:, 1, 0], np.linspace(0.5, 0.95, 10))
    assert 0.8999999999999999 in mo[:, 0, 0] and 0.9 not in mo[:, 0, 0]
    assert 0.44999999999999996 in mo[:, 2, 1] and 0.6499999999999999 in mo[:, 2, 2]


def _perturbed_sets(dts, n, seed=3):
    """n detection sets on the same frames: the given detections with jittered scores and dropped rows."""
    rng = np.random.default_rng(seed)
    sets = []
    for _ in range(n):
        s = []
        for d in dts:
            keep = rng.uniform(size=len(d["name"])) < 0.85
            e = {k: np.asarray(v)[keep] for k, v in d.items()}
            e["score"] = np.clip(e["score"] + rng.normal(0, 0.05, len(e["score"])), 0.0, 1.0)
            s.append(e)
        sets.append(s)
    return sets


def test_k_set_evaluation_equals_single_calls_on_the_host():
    (gts, dts), _ = _gold()
    sets = _perturbed_sets(dts, 3)
    many = K.coco_eval_many(gts, sets, [0, 1, 2], overlap_fn=O.rotate_iou_eval)
    both = K.eval_many(gts, sets, [0, 1, 2], (11, 40, "coco"), overlap_fn=O.rotate_iou_eval)
    for s, d in enumerate(sets):
        one = K.coco_eval(gts, d, [0, 1, 2], overlap_fn=O.rotate_iou_eval)
        _same_tables({"coco": many[s]}, {"coco": one})
        want = {rp: K.official_eval(gts, d, [0, 1, 2], overlap_fn=O.rotate_iou_eval, recall_positions=rp)
                for rp in (11, 40)}
        want["coco"] = one
        _same_tables(both[s], want)


def test_argument_errors():
    (gts, dts), _ = _gold()
    for bad in ((), (11, "voc"), (41,)):
        with pytest.raises(ValueError, match="tables"):
            K.eval_many(gts, [dts], [0], bad, overlap_fn=O.rotate_iou_eval)
    with pytest.raises(KeyError):
        K.coco_eval(gts, dts, ["Truck"], overlap_fn=O.rotate_iou_eval)
    from sassd_b200 import test as T
    base = ["c.py", "a.pth"]
    assert T.parse_args(base + ["--data-root", "r", "--coco"]).coco
    for bad in (["--data-root", "r", "--split", "test", "--out", "o", "--coco"], ["--drive", "d", "--out", "o", "--coco"]):
        with pytest.raises(SystemExit):
            T.parse_args(base + bad)


def test_device_abi_refuses_bad_arguments():
    """The C ABI checks its counts before touching the device."""
    from sassd_b200 import lib as L
    lib = L.load()
    args = [None] * 6 + [0, None]
    for fields in (dict(nsets=0), dict(nframes=-1), dict(nclass=0), dict(ndiff=0), dict(nover=0), dict(max_nd=-1),
                   dict(nsets=1000, nclass=8, ndiff=3, nover=10000)):     # the last: past 2^31 (job, threshold) items
        d = L.KittiEvalDesc(nsets=1, nframes=1, nclass=1, ndiff=1, nover=1)
        for k, v in fields.items():
            setattr(d, k, v)
        assert lib.sassd_kitti_eval_match(ctypes.byref(d), *args) == -1, fields
    assert lib.sassd_kitti_eval_flags(-1, *([None] * 4), 0, None, None, 1, None, 1, None, None, None, None, None) == -1
    assert lib.sassd_kitti_eval_overlaps(0, 1, *([None] * 9), 0, None, None, None, None) == -1
    assert lib.sassd_kitti_aos_table(1, -1, *([None] * 6)) == -1
    assert lib.sassd_kitti_eval_workspace_bytes(-1, 0) == 0


def test_aos_table_uses_the_host_matchers_cos():
    from sassd_b200 import lib as L
    rng = np.random.default_rng(0)
    ng, nd = np.array([3, 0, 5]), np.array([4, 2, 0, 1, 1, 7])        # 2 sets x 3 frames
    gt_off, dt_off = K._offsets(ng), K._offsets(nd)
    ov_off = K._offsets(nd * np.tile(ng, 2), np.int64)
    ga, da = rng.uniform(-np.pi, np.pi, ng.sum()), rng.uniform(-np.pi, np.pi, nd.sum())
    out = np.zeros((int(ov_off[-1]),))
    L.check(L.load().sassd_kitti_aos_table(2, 3, K._p(gt_off), K._p(dt_off), K._p(ov_off), K._p(ga), K._p(da),
                                           K._p(out)), "aos table")
    for b in range(6):
        f = b % 3
        blk = out[ov_off[b]:ov_off[b + 1]].reshape(nd[b], ng[f])
        for j in range(nd[b]):
            for i in range(ng[f]):
                assert blk[j, i] == (1.0 + math.cos(ga[gt_off[f] + i] - da[dt_off[b] + j])) / 2.0


# ------------------------------------------------------------------------------------------------------------ GPU
def _device_overlaps(boxes, query, criterion):
    """The product's CUDA rotated overlaps, one launch per call: the host path then differs from the device path in
    cleaning and matching only."""
    return K.rotate_iou_gpu_eval(boxes, query, criterion)


def _hard_sets(nsets, nframes=60, seed=11):
    """GT and nsets detection sets with the cases the matcher has edges at."""
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden_eval import synth_annos
    rng = np.random.default_rng(seed)
    gts, dts = synth_annos(rng, nframes)
    sets = _perturbed_sets(dts, nsets, seed + 1)

    def frame(names, bboxes, scores=None, alpha=None):
        n = len(names)
        bb = np.asarray(bboxes, np.float64).reshape(n, 4)
        loc = np.stack([np.linspace(-5, 5, n), np.full(n, 1.6), np.full(n, 20.0)], 1) if n else np.zeros((0, 3))
        a = dict(name=np.array(names, dtype=str).reshape(n), truncated=np.zeros(n), occluded=np.zeros(n, np.int64),
                 alpha=np.zeros(n) if alpha is None else np.asarray(alpha, np.float64), bbox=bb,
                 dimensions=np.tile([3.9, 1.56, 1.6], (n, 1)), location=loc, rotation_y=np.zeros(n))
        if scores is not None:
            a["score"] = np.asarray(scores, np.float64)
        return a
    box = [0.0, 0.0, 100.0, 100.0]
    # 2-D IoU exactly 0.65 (> 0.6499999999999999 of Cyclist's linspace) and 0.9 (> Car's 0.8999999999999999)
    extra = [
        (frame([], []), frame(["Car"], [box], [0.9])),                                      # no GT
        (frame(["Car", "Pedestrian"], [box, [200, 0, 260, 120]]), frame([], [], [])),      # no detections
        (frame(["DontCare", "DontCare"], [box, [300, 0, 400, 80]]),                         # only DontCare
         frame(["Car", "Car"], [[0, 0, 100, 90], [310, 0, 390, 70]], [0.7, 0.6])),
        (frame(["Cyclist", "Cyclist"], [box, [200, 0, 300, 100]]),
         frame(["Cyclist", "Cyclist"], [[0, 0, 100, 65], [200, 0, 300, 65]], [0.5, 0.5])),  # tied scores
        (frame(["Car"], [box]), frame(["Car", "Car"], [[0, 0, 100, 90], [0, 0, 100, 65]], [0.5, 0.5])),
        (frame(["Car"] * 6, [[150 * i, 0, 150 * i + 100, 100] for i in range(6)]),        # > 128 detections
         frame(["Car"] * 150, [[7 * i, 0, 7 * i + 100, 90 + (i % 11)] for i in range(150)],
               np.round(np.linspace(0.1, 0.95, 150), 2), np.linspace(-3, 3, 150))),
    ]
    rng2 = np.random.default_rng(seed + 2)
    for g, d in extra:
        gts.append(g)
        for s in sets:
            e = copy.deepcopy(d)
            e["score"] = np.clip(e["score"] + np.round(rng2.normal(0, 0.02, len(e["score"])), 2), 0, 1)
            s.append(e)
    return gts, sets


@pytest.mark.gpu
def test_device_evaluator_equals_the_goldens():
    (gts, dts), gold = _gold()
    for tag, classes in CLASS_SETS:
        _same_coco(K.coco_eval(gts, dts, classes), gold, tag)
    assert K.get_coco_eval_result(gts, dts, [0, 1, 2]) == str(gold["text_c012"])
    g = np.load(GOLD)
    text, ap = K.official_eval(gts, dts, [0, 1, 2])
    assert text == str(g["official_text"]) and K.get_official_eval_result(gts, dts, [0, 1, 2]) == text
    for k, kk in (("bbox", "ap_bbox"), ("bev", "ap_bev"), ("d3", "ap_d3"), ("aos", "ap_aos")):
        np.testing.assert_array_equal(ap[k], g[kk])
    r = np.load(os.path.join(HERE, "golden", "eval_r40.npz"))
    _, ap40 = K.official_eval(gts, dts, [0, 1, 2], recall_positions=40)
    for k, p in (("bbox", "prec_0"), ("bev", "prec_1"), ("d3", "prec_2"), ("aos", "orient_0")):
        np.testing.assert_array_equal(ap40[k], K.get_mAP_R40(r[p]), err_msg=k)


@pytest.mark.gpu
@pytest.mark.parametrize("nsets", [1, 4, 10])
def test_device_evaluator_equals_the_host_path_bit_for_bit(nsets):
    gts, sets = _hard_sets(nsets)
    assert max(len(d["name"]) for s in sets for d in s) > 128
    for classes in ([0, 1, 2], [2]):
        mo = np.concatenate([np.stack([K.OVERLAP_0_7, K.OVERLAP_0_5])[:, :, classes], K.coco_min_overlaps(classes)])
        aos = [K._aos_flag(s) for s in sets]
        dev = K._eval_device(gts, sets, classes, [0, 1, 2], mo, aos)
        for metric in (0, 1, 2):
            host = K.eval_class_many(gts, sets, classes, [0, 1, 2], metric, mo,
                                     aos if metric == 0 else [False] * nsets, _device_overlaps)
            for s in range(nsets):
                for key in ("precision", "recall", "orientation"):
                    np.testing.assert_array_equal(dev[metric][s][key], host[s][key],
                                                  err_msg="classes %s metric %d set %d %s" % (classes, metric, s, key))
        got = K.eval_many(gts, sets, classes, (11, 40, "coco"))
        want = K.eval_many(gts, sets, classes, (11, 40, "coco"), overlap_fn=_device_overlaps)
        for a, b in zip(got, want):
            _same_tables(a, b)


@pytest.mark.gpu
def test_driver_prints_coco_tables_alone_and_for_a_sweep(tmp_path):
    import json
    from sassd_b200 import checkpoint
    from sassd_b200 import test as T
    from tests.checkpoint_weights import CAR_CFG, checkpoint_state_dict
    from tests.kitti_root import write_tree
    root = str(tmp_path / "kitti")
    write_tree(root)
    ckpts = []
    for seed in (1, 2):
        ckpts.append(str(tmp_path / ("epoch_%d.pth" % seed)))
        checkpoint.save_checkpoint(checkpoint_state_dict(seed), ckpts[-1])
    base = ["--data-root", root, "--split", "trainval", "--lidar", "velodyne", "--batch", "4", "--workers", "2",
            "--r40", "--coco"]
    singles = []
    for i, c in enumerate(ckpts):
        printed = []
        res = T.run(T.parse_args([CAR_CFG, c, "--json", str(tmp_path / ("single_%d.json" % i))] + base),
                    log=lambda *a, **k: printed.append(" ".join(str(x) for x in a)))
        assert res["text_coco"].startswith("Car coco AP@0.50:0.05:0.95:\n")
        assert printed.index(res["text"]) < printed.index(res["text_r40"]) < printed.index(res["text_coco"])
        with open(str(tmp_path / ("single_%d.json" % i))) as fh:
            assert json.load(fh)["ap_coco"] == res["ap_coco"]
        singles.append(res)
    printed = []
    res = T.run(T.parse_args([CAR_CFG, ckpts[0], "--checkpoints", ckpts[1], "--json", str(tmp_path / "sweep.json")]
                             + base), log=lambda *a, **k: printed.append(" ".join(str(x) for x in a)))
    for e, single in zip(res["checkpoints"], singles):
        for key in ("text", "ap", "text_r40", "ap_r40", "text_coco", "ap_coco"):
            assert e[key] == single[key], key
        assert single["text_coco"] in printed
    summary = printed[printed.index("summary: 2 checkpoints (moderate 3D AP)") + 1:]
    assert all("R40" in s and "COCO" in s for s in summary[:2])
    for s, single in zip(summary, singles):
        assert "COCO %6.2f" % single["ap_coco"]["d3"][0][1] in s

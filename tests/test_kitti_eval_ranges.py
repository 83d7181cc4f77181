"""KITTI AP per range bin and the per-object match table (kitti_eval.eval_many(ranges=...), match_table, tp_errors).

* CPU: the host path (the oracle's rotated overlaps injected) equals the reference's BEV / 3-D precision and AP of
  every bin (tests/golden/eval_ranges.npz, make_golden_eval_ranges.py: the unmodified reference on annotations
  transformed to the bin's semantics), and the match table's state counts equal the reference's compute_statistics_jit
  (tp, fp, fn).  ranges=[0, inf] reproduces the whole-range arrays; a partition's bins sum to the whole range's valid
  GT; TP errors follow their formulas; bad edges are refused by the API and both commands.
* GPU: the device path equals the goldens and equals the host path bit for bit (range APs, flags, ranges, match table,
  TP errors) at K = 1 and 3 sets with NaN locations and objects on the edges; both commands with --ranges / --matches,
  each checkpoint of a sweep giving what a run of its own gives.
"""
import copy
import json
import math
import os

import numpy as np
import pytest

from oracle import kitti_eval as O
from sassd_b200 import kitti_eval as K
from sassd_b200 import lib as L
from tests.test_kitti_eval import KEYS

HERE = os.path.dirname(os.path.abspath(__file__))
RANGES_GOLD = os.path.join(HERE, "golden", "eval_ranges.npz")
TABLES = (11, 40, "coco")
OVERLAP = np.stack([K.OVERLAP_0_7, K.OVERLAP_0_5])


def _gold():
    g = np.load(RANGES_GOLD)
    n = int(g["nframes"])
    gts = [{k: g["gt%d_%s" % (i, k)] for k in KEYS} for i in range(n)]
    dts = [{k: g["dt%d_%s" % (i, k)] for k in KEYS + ("score",)} for i in range(n)]
    return gts, dts, g


def _bins(edges):
    return list(zip(edges[:-1], edges[1:]))


def _same_ap(a, b, what):
    for k in ("bbox", "bev", "d3", "aos"):
        if a[k] is None or b[k] is None:
            assert a[k] is None and b[k] is None, (what, k)
        else:
            np.testing.assert_array_equal(a[k], b[k], err_msg="%s %s" % (what, k))


def _same_eval(a, b):
    """Two eval_many dicts equal bit for bit: tables, range tables and match tables."""
    assert a.keys() == b.keys()
    for t in (t for t in a if t in TABLES):
        assert a[t][0] == b[t][0]
        _same_ap(a[t][1], b[t][1], t)
    if "ranges" in a:
        assert len(a["ranges"]) == len(b["ranges"])
        for (lo, hi, ra), (lo2, hi2, rb) in zip(a["ranges"], b["ranges"]):
            assert (lo, hi) == (lo2, hi2) and ra.keys() == rb.keys()
            for t in ra:
                assert ra[t][0] == rb[t][0], (lo, t)
                _same_ap(ra[t][1], rb[t][1], "%s %s" % (lo, t))
    if "matches" in a:
        _same_table(a["matches"], b["matches"])


def _same_table(a, b):
    assert a.keys() == b.keys()
    for k in a:
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape, k
        assert x.tobytes() == y.tobytes(), k


def _counts(table, ci, di, m):
    """(tp, fp, fn) of a match table's (class, difficulty, metric)."""
    st = table["dt_state"][ci, di, m]
    fn = (table["gt_flag"][ci, di] == 0) & (table["gt_det"][ci, di, m] == -1)
    return int((st == L.KITTI_DT_TP).sum()), int((st == L.KITTI_DT_FP).sum()), int(fn.sum())


def _check_against_gold(evaluate_prec, evaluate_many, table):
    """evaluate_prec(classes, diffs, metric, min_overlaps, bins) -> precision [C, entries, M, 41]."""
    gts, dts, g = _gold()
    edges = tuple(g["edges"])
    bins = _bins(edges)
    for c in (0, 1, 2):
        for metric in (1, 2):
            prec = evaluate_prec([c], [0, 1, 2] * len(bins), metric, OVERLAP[:, :, [c]],
                                 [b for b in bins for _ in range(3)])
            for bi in range(len(bins)):
                np.testing.assert_array_equal(prec[:, 3 * bi:3 * bi + 3], g["prec_c%d_b%d_m%d" % (c, bi, metric)],
                                              err_msg="class %d bin %d metric %d" % (c, bi, metric))
    ev = evaluate_many(gts, [dts], [0, 1, 2], (11,), edges)[0]
    for bi, (lo, hi, res) in enumerate(ev["ranges"]):
        assert (lo, hi) == bins[bi]
        for c in (0, 1, 2):
            for metric, key in ((1, "bev"), (2, "d3")):
                np.testing.assert_array_equal(res[11][1][key][c], g["ap_c%d_b%d_m%d" % (c, bi, metric)][0])
    assert not any(g["ap_c%d_b0_m%d" % (c, m)].any() for c in (0, 1, 2) for m in (1, 2))   # the empty bin: AP 0
    for ci in range(3):
        for di in range(3):
            for m in range(3):
                assert _counts(table, ci, di, m) == tuple(g["stat_c%d_d%d_m%d" % (ci, di, m)]), (ci, di, m)


# ------------------------------------------------------------------------------------------------------------ CPU
def test_golden_has_objects_on_an_edge_and_across_edges():
    gts, dts, g = _gold()
    r = np.concatenate([K.ground_range(a) for a in gts])
    assert 20.0 in r and (r < 4).sum() == 0
    edges = g["edges"]
    assert edges[-1] == np.inf and len(edges) == 5
    for lo, hi in _bins(edges)[1:]:
        assert ((lo <= r) & (r < hi)).sum() > 0


def test_host_path_equals_the_reference_per_range_bin():
    gts, dts, _ = _gold()

    def prec(classes, diffs, metric, mo, bins):
        return K.eval_class_many(gts, [dts], classes, diffs, metric, mo, [False], O.rotate_iou_eval, None,
                                 bins)[0]["precision"]

    def many(gts, sets, classes, tables, ranges):
        return K.eval_many(gts, sets, classes, tables, O.rotate_iou_eval, ranges=ranges)
    _check_against_gold(prec, many, K.match_table(gts, [dts], [0, 1, 2], overlap_fn=O.rotate_iou_eval)[0])


def test_whole_range_bin_reproduces_the_whole_range_on_the_host():
    gts, dts, _ = _gold()
    sets = [dts, [dict(d, score=np.clip(d["score"] - 0.1, 0, 1)) for d in dts]]
    ev = K.eval_many(gts, sets, [0, 1, 2], TABLES, O.rotate_iou_eval, ranges=[0, np.inf])
    base = K.eval_many(gts, sets, [0, 1, 2], TABLES, O.rotate_iou_eval)
    for e, b in zip(ev, base):
        assert "ranges" not in b and "matches" not in b
        (lo, hi, res), = e["ranges"]
        assert (lo, hi) == (0.0, np.inf)
        for t in TABLES:
            assert e[t][0] == b[t][0]
            _same_ap(res[t][1], b[t][1], t)
            assert res[t][0] != b[t][0] and " range [0, inf) m:" in res[t][0]
    assert "Car AP@0.70, 0.70, 0.70 range [0, inf) m:\n" in ev[0]["ranges"][0][2][11][0]
    assert "Car coco AP@0.50:0.05:0.95 range [0, inf) m:\n" in ev[0]["ranges"][0][2]["coco"][0]


def test_bins_of_a_partition_sum_to_the_whole_range():
    gts, dts, g = _gold()
    for edges in (tuple(g["edges"]), (0, 7.5, 20.0, 20.5, 33, np.inf)):
        for c in (0, 1, 2):
            for d in (0, 1, 2):
                whole = K._GtSide(gts, c, d).total_valid
                assert whole == sum(K._GtSide(gts, c, d, b).total_valid for b in _bins(edges))
                assert whole > 0


def test_detections_across_an_edge_are_neither_tp_nor_fp_nor_fn():
    """A detection just outside a bin matching a GT just inside it: in the GT's bin it is no TP and the GT no FN; in the
    detection's bin it is no FP."""
    def anno(z, score=None):
        h = 720 * 1.56 / z
        a = dict(name=np.array(["Car"]), truncated=np.zeros(1), occluded=np.zeros(1, np.int64), alpha=np.zeros(1),
                 bbox=np.array([[600.0, 190 - h / 2, 600 + 720 * 3.9 / z, 190 + h / 2]]),
                 dimensions=np.array([[3.9, 1.56, 1.6]]), location=np.array([[0.0, 1.6, z]]), rotation_y=np.zeros(1))
        if score is not None:
            a["score"] = np.array([score])
        return a
    gts, dts = [anno(19.95)], [anno(20.05, 0.9)]
    for lo, hi in ((0, 20), (20, 40)):
        gs = K._GtSide(gts, 0, 0, (lo, hi))
        ov = K.calculate_overlaps(gts, dts, 2, O.rotate_iou_eval)
        packed = K._Packed(gs, dts, ov, 0, 0, (lo, hi))
        assert packed.match(2, 0.5, [0.0])[0][0, :3].tolist() == [0, 0, 0]
        assert gs.total_valid == (1 if lo == 0 else 0)
    ev = K.eval_many(gts, [dts], [0], (11,), O.rotate_iou_eval, ranges=[0, 20, 40])[0]
    assert ev[11][1]["d3"][0, 0, 1] == 100.0 / 11       # one TP: only the first of the 11 recall samples
    assert [r[2][11][1]["d3"][0, 0, 1] for r in ev["ranges"]] == [0.0, 0.0]


def test_tp_errors_follow_their_formulas():
    gts, dts, _ = _gold()
    table = K.match_table(gts, [dts], [0, 1, 2], overlap_fn=O.rotate_iou_eval)[0]
    gcam, dcam = K._flat_cam(gts), K._flat_cam(dts)
    n = 0
    for ci in range(3):
        for di in range(3):
            j = table["gt_det"][ci, di, 2]
            err = table["tp_errors"][ci, di]
            for i in range(len(j)):
                if j[i] < 0 or table["dt_state"][ci, di, 2][j[i]] != L.KITTI_DT_TP:
                    assert np.isnan(err[i]).all()
                    continue
                gq, dq = gcam[i], dcam[j[i]]
                vi = min(gq[3], dq[3]) * min(gq[4], dq[4]) * min(gq[5], dq[5])
                vg, vd = gq[3] * gq[4] * gq[5], dq[3] * dq[4] * dq[5]
                dr = (dq[6] - gq[6]) % (2 * math.pi)
                want = [math.hypot(dq[0] - gq[0], dq[2] - gq[2]), 1 - vi / (vg + vd - vi), min(dr, 2 * math.pi - dr)]
                np.testing.assert_allclose(err[i], want, rtol=1e-12, atol=1e-12)
                assert 0 <= err[i, 2] <= np.pi and 0 <= err[i, 1] < 1
                n += 1
    assert n > 50
    rows = np.array([[1.0, 1.6, 10.0, 3.9, 1.5, 1.6, 0.3], [-4.0, 1.6, 30.0, 0.8, 1.7, 0.6, -3.1]])
    np.testing.assert_array_equal(K.tp_errors(rows, rows), np.zeros((2, 3)))
    wrap = K.tp_errors(np.tile(rows[:1], (5, 1)), rows[:1] + np.array([[0, 0, 0, 0, 0, 0, a] for a in (
        np.pi, -np.pi, 3 * np.pi, 2 * np.pi - 1e-15, -7.0)]))[:, 2]
    assert np.all((0 <= wrap) & (wrap <= np.pi))
    np.testing.assert_allclose(wrap, [np.pi, np.pi, np.pi, 0, 7.0 - 2 * np.pi], atol=1e-12)


def test_match_table_layout_and_summary():
    gts, dts, g = _gold()
    table = K.match_table(gts, [dts], ["Car", "Pedestrian"], overlap_fn=O.rotate_iou_eval)[0]
    G, D = sum(len(a["name"]) for a in gts), sum(len(a["name"]) for a in dts)
    assert table["gt_det"].shape == (2, 3, 3, G) and table["dt_state"].shape == (2, 3, 3, D)
    assert table["tp_errors"].shape == (2, 3, G, 3) and table["gt_flag"].shape == (2, 3, G)
    np.testing.assert_array_equal(table["gt_range"], np.concatenate([K.ground_range(a) for a in gts]))
    assert table["dt_off"][-1] == D and table["gt_off"][-1] == G
    # a matched pair's overlap is the metric's, above the min overlap
    ov = K.calculate_overlaps(gts, dts, 1, O.rotate_iou_eval)
    for f in range(len(gts)):
        g0, d0 = table["gt_off"][f], table["dt_off"][f]
        for i in range(table["gt_off"][f + 1] - g0):
            j = table["gt_det"][0, 1, 1, g0 + i]
            if j >= 0:
                assert table["gt_overlap"][0, 1, 1, g0 + i] == ov[f][j - d0, i] > 0.7
            else:
                assert table["gt_overlap"][0, 1, 1, g0 + i] == 0
    summary = K.tp_error_summary(table, ["Car", "Pedestrian"], ranges=g["edges"])
    for ci, s in enumerate(summary):
        tp = np.flatnonzero(~np.isnan(table["tp_errors"][ci, 1, :, 0]))
        assert s["tp"] == len(tp) == _counts(table, ci, 1, 2)[0]
        assert s["ate"] == np.mean(table["tp_errors"][ci, 1, tp, 0])
        assert sum(b["tp"] for b in s["ranges"]) == s["tp"] and s["ranges"][0]["ate"] is None
        assert s["ranges"][-1]["hi"] is None
    json.dumps(summary)


@pytest.mark.parametrize("bad", [[0], [], [0, 0], [10, 5], [-1, 5], [0, np.nan], [0, np.inf, np.inf], ["a", "b"]])
def test_bad_edges_are_refused(bad, tmp_path, capsys):
    gts, dts, _ = _gold()
    with pytest.raises(ValueError, match="ranges"):
        K.eval_many(gts[:3], [dts[:3]], [0], (11,), O.rotate_iou_eval, ranges=bad)
    if not bad or isinstance(bad[0], str):
        return
    root = str(tmp_path)
    os.makedirs(os.path.join(root, "ImageSets"))
    os.makedirs(os.path.join(root, "training", "label_2"))
    open(os.path.join(root, "ImageSets", "val.txt"), "w").close()
    edges = [repr(float(e)) for e in bad]
    with pytest.raises(SystemExit) as e:
        K.parse_args(["--data-root", root, "--results", root, "--ranges"] + edges)
    assert e.value.code == 2 and "--ranges" in capsys.readouterr().err
    from sassd_b200 import test as T
    with pytest.raises(SystemExit) as e:
        T.parse_args(["c.py", "a.pth", "--data-root", root, "--ranges"] + edges)
    assert e.value.code == 2 and "--ranges" in capsys.readouterr().err


def test_command_arguments():
    from sassd_b200 import test as T
    a = T.parse_args(["c.py", "a.pth", "--data-root", "r", "--ranges", "0", "20", "inf", "--matches", "m.npz"])
    assert a.ranges == [0.0, 20.0, np.inf] and a.matches == "m.npz"
    assert T.parse_args(["c.py", "a.pth", "--data-root", "r"]).ranges is None
    for bad in (["--split", "test", "--out", "o", "--ranges", "0", "20"], ["--split", "test", "--out", "o", "--matches",
                                                                          "m.npz"]):
        with pytest.raises(SystemExit):
            T.parse_args(["c.py", "a.pth", "--data-root", "r"] + bad)


def test_device_abi_refuses_bad_arguments():
    lib = L.load()
    assert lib.sassd_kitti_eval_flags_ranged(-1, *([None] * 5), 0, *([None] * 3), 1, None, 1, *([None] * 8)) == -1
    d = L.KittiEvalDesc(nsets=1, nframes=1, nclass=1, ndiff=1, nover=1)
    for row, ndiff in ((1, 1), (-1, 1), (0, 0), (0, 2)):
        assert lib.sassd_kitti_eval_assign(K.ctypes.byref(d), row, ndiff, *([None] * 7), 0, None) == -1


# ------------------------------------------------------------------------------------------------------------ GPU
def _device_overlaps(boxes, query, criterion):
    return K.rotate_iou_gpu_eval(boxes, query, criterion)


def _edge_sets(nsets, seed=5):
    """The golden's annotations, nsets perturbed detection sets, and a frame with NaN locations and objects on the
    edges (20 m exactly, just either side of 40 m)."""
    from tests.test_kitti_eval_coco import _perturbed_sets
    gts, dts, g = _gold()
    sets = _perturbed_sets(dts, nsets, seed)
    gt = copy.deepcopy(gts[-4])
    gt["location"] = gt["location"].copy()
    gt["location"][1] = [np.nan, 1.6, 30.0]
    gts = gts + [gt]
    for s in sets:
        d = copy.deepcopy(dts[-4])
        d["location"] = d["location"].copy()
        d["location"][2] = [np.nan, 1.6, np.nan]
        s.append(d)
    return gts, sets, tuple(g["edges"])


@pytest.mark.gpu
def test_device_path_equals_the_reference_per_range_bin():
    gts, dts, _ = _gold()

    def prec(classes, diffs, metric, mo, bins):
        return K._eval_device_full(gts, [dts], classes, diffs, mo, [False], bins)[0][metric][0]["precision"]

    def many(gts, sets, classes, tables, ranges):
        return K.eval_many(gts, sets, classes, tables, ranges=ranges)
    _check_against_gold(prec, many, K.match_table(gts, [dts], [0, 1, 2])[0])


@pytest.mark.gpu
@pytest.mark.parametrize("nsets", [1, 3])
def test_device_equals_host_bit_for_bit(nsets):
    gts, sets, edges = _edge_sets(nsets)
    for classes in ([0, 1, 2], [1]):
        dev = K.eval_many(gts, sets, classes, TABLES, ranges=edges, match=True)
        host = K.eval_many(gts, sets, classes, TABLES, _device_overlaps, ranges=edges, match=True)
        for a, b in zip(dev, host):
            _same_eval(a, b)
        assert np.isnan(dev[0]["matches"]["gt_range"]).sum() == 1
        assert np.isnan(dev[-1]["matches"]["dt_range"]).sum() == 1
    tables = K.match_table(gts, sets, [0, 1, 2], (1,))
    assert tables[0]["gt_det"].shape[1] == 1
    for a, b in zip(tables, K.match_table(gts, sets, [0, 1, 2], (1,), _device_overlaps)):
        _same_table(a, b)
    # the whole-range bin reproduces the whole range on the device (no NaN locations there)
    gts0, dts0, _ = _gold()
    ev = K.eval_many(gts0, [dts0], [0, 1, 2], TABLES, ranges=[0, np.inf])[0]
    for t in TABLES:
        _same_ap(ev["ranges"][0][2][t][1], ev[t][1], t)


@pytest.mark.gpu
def test_ranged_flags_without_ranges_are_the_flags():
    import torch
    from sassd_b200 import ops
    gts, sets, edges = _edge_sets(1)
    gt, dt = K.AnnoBlock.from_annos(gts), K.AnnoBlock.from_annos(sets[0])
    cls = torch.tensor([[0, 3], [1, 4], [2, -1]], dtype=torch.int32, device="cuda")
    lim = torch.tensor([[0, 0.15, 40], [1, 0.3, 25], [2, 0.5, 25]], dtype=torch.float64, device="cuda")
    base = ops.kitti_eval_flags(gt.name_id, gt.occluded, gt.truncated, gt.bbox, dt.name_id, dt.bbox, cls, lim)
    ranged = ops.kitti_eval_flags_ranged(gt.name_id, gt.occluded, gt.truncated, gt.bbox, gt.cam, dt.name_id, dt.bbox,
                                         dt.cam, cls, lim, None)
    for a, b in zip(base, ranged):
        assert torch.equal(a, b)
    r = ranged[3].cpu().numpy()
    np.testing.assert_array_equal(r, np.concatenate([K.ground_range(a) for a in gts]))
    # a partition's bins sum to the whole range's valid GT (no NaN GT of a class here: the NaN row is not counted)
    bins = torch.tensor([[lo, hi] for lo, hi in _bins(edges) for _ in range(3)], dtype=torch.float64, device="cuda")
    part = ops.kitti_eval_flags_ranged(gt.name_id, gt.occluded, gt.truncated, gt.bbox, gt.cam, dt.name_id, dt.bbox,
                                       dt.cam, cls, lim.repeat(len(bins) // 3, 1), bins)[2].cpu().numpy()
    whole = base[2].cpu().numpy()
    nan_valid = np.isnan(r)[None, None, :] & (base[0].cpu().numpy() == 0)
    assert (part.reshape(3, -1, 3).sum(1) + nan_valid.sum(-1) == whole).all()


def _write_dirs(tmp, gts, sets, ids):
    from tests.test_kitti_eval_dirs import _write_sets
    return _write_sets(tmp, gts, sets, ids)


@pytest.mark.gpu
def test_eval_command_with_ranges_and_matches(tmp_path):
    from sassd_b200 import kitti_data as KD
    from sassd_b200 import test as T
    from tests.kitti_root import write_tree
    root = str(tmp_path / "kitti")
    write_tree(root)
    ids = KD.read_split(root, "trainval")
    gt = KD.read_labels(os.path.join(root, "training", "label_2"), ids)
    from tests.test_kitti_eval_coco import _perturbed_sets
    sets = _perturbed_sets([dict({k: g[k] for k in KEYS}, score=np.linspace(0.2, 0.9, len(g["name"]))) for g in gt], 2,
                           seed=9)
    dirs = []
    for k, s in enumerate(sets):
        dirs.append(str(tmp_path / ("set%d" % k)))
        T.write_results(dirs[-1], ids, [dict(a, dimensions=np.asarray(a["dimensions"], np.float64)) for a in s])
    js, mz = str(tmp_path / "e.json"), str(tmp_path / "m.npz")
    printed = []
    res = K.main(["--data-root", root, "--split", "trainval", "--results"] + dirs + ["--classes", "Car", "Pedestrian",
                 "--r40", "--ranges", "0", "20", "inf", "--matches", mz, "--json", js],
                 log=lambda *a, **k: printed.append(" ".join(a)))
    want = K.eval_many(KD.read_labels(os.path.join(root, "training", "label_2"), ids),
                       [KD.read_labels(d, ids) for d in dirs], ["Car", "Pedestrian"], (11, 40), ranges=[0, 20, np.inf],
                       match=True)
    z = np.load(mz)
    assert list(z["labels"]) == dirs
    for k, (w, e) in enumerate(zip(want, res["results"])):
        assert e["text_ranges"] == [r[2][11][0] for r in w["ranges"]]
        assert e["text_ranges_r40"] == [r[2][40][0] for r in w["ranges"]]
        assert e["ap_ranges"][1] == dict(lo=20.0, hi=None, ap=K.ap_lists(w["ranges"][1][2][11][1]))
        assert e["tp_errors"] == K.tp_error_summary(w["matches"], ["Car", "Pedestrian"], ranges=[0, 20, np.inf])
        for name, v in w["matches"].items():
            np.testing.assert_array_equal(z["set%d_%s" % (k, name)], v)
        at = printed.index("== %s ==" % dirs[k])
        assert printed[at + 1:at + 3] == [w[11][0], w[40][0]]
        assert printed[at + 3:at + 7] == [w["ranges"][0][2][11][0], w["ranges"][1][2][11][0],
                                          w["ranges"][0][2][40][0], w["ranges"][1][2][40][0]]
    line = printed[printed.index("summary: 2 directories (moderate 3D AP)") + 1]
    assert "Car 3d mod [20, inf) R11 %6.2f R40" % want[0]["ranges"][1][2][11][1]["d3"][0, 1, 0] in line
    assert "Pedestrian TP %d ATE" % res["results"][0]["tp_errors"][1]["tp"] in line
    with open(js) as fh:
        assert json.load(fh)["results"][1]["ap_ranges_r40"] == res["results"][1]["ap_ranges_r40"]
    # without the new options: the same tables and no new keys
    plain = K.main(["--data-root", root, "--split", "trainval", "--results"] + dirs + ["--classes", "Car", "Pedestrian",
                   "--r40"], log=lambda *a, **k: None)
    for e, p in zip(res["results"], plain["results"]):
        assert set(e) - set(p) == {"text_ranges", "ap_ranges", "text_ranges_r40", "ap_ranges_r40", "tp_errors"}
        assert all(e[k] == p[k] for k in p)


@pytest.mark.gpu
def test_driver_ranges_for_a_sweep_equal_single_runs(tmp_path):
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
            "--coco", "--ranges", "0", "15", "30", "inf"]
    singles = []
    for i, c in enumerate(ckpts):
        printed = []
        res = T.run(T.parse_args([CAR_CFG, c, "--matches", str(tmp_path / ("single_%d.npz" % i))] + base),
                    log=lambda *a, **k: printed.append(" ".join(str(x) for x in a)))
        assert len(res["text_ranges"]) == 3 and len(res["text_ranges_coco"]) == 3
        assert printed.index(res["text_coco"]) < printed.index(res["text_ranges"][0])
        assert any(p.startswith("summary: Car 3d mod [0, 15) R11") for p in printed)
        singles.append(res)
    printed = []
    res = T.run(T.parse_args([CAR_CFG, ckpts[0], "--checkpoints", ckpts[1], "--matches", str(tmp_path / "sweep.npz")]
                             + base), log=lambda *a, **k: printed.append(" ".join(str(x) for x in a)))
    sweep = np.load(str(tmp_path / "sweep.npz"))
    for k, (e, single) in enumerate(zip(res["checkpoints"], singles)):
        for key in ("text", "ap", "text_coco", "ap_coco", "text_ranges", "ap_ranges", "text_ranges_coco",
                    "ap_ranges_coco", "tp_errors"):
            assert e[key] == single[key], key
        one = np.load(str(tmp_path / ("single_%d.npz" % k)))
        for name in one.files:
            if name.startswith("set0_"):
                np.testing.assert_array_equal(sweep["set%d_%s" % (k, name[5:])], one[name])
    summary = printed[printed.index("summary: 2 checkpoints (moderate 3D AP)") + 1:]
    assert all("Car 3d mod [15, 30) R11" in s and "Car TP " in s for s in summary[:2])

"""Bootstrap replicates of the KITTI AP (kitti_eval.eval_many(bootstrap=...), bootstrap_indices, percentile_interval,
paired_summary, --bootstrap of both commands).

* CPU: the host path (the oracle's rotated overlaps injected) equals the unmodified reference on each replicate's
  resampled lists (tests/golden/eval_bootstrap.npz, make_golden_eval_bootstrap.py: seeded rows, the identity, one
  frame repeated, a draw without Pedestrian GT); the identity row is eval_many's AP; a set against itself differs by 0;
  the indices are deterministic per row; bad indices and options are refused; the helpers are numpy's; the [R, ...]
  numpy tail equals the per-replicate one.
* GPU: the device path equals the host path bit for bit (K = 1 and 3, every table, with and without ranges, NaN
  locations and scores, several replicate chunks), and each of 16 replicates of 3769 synthetic frames equals eval_many
  on its lists; both commands with --bootstrap keep their tables and give a sweep's checkpoints their single runs'
  intervals.
"""
import copy
import json
import os

import numpy as np
import pytest

from oracle import kitti_eval as O
from sassd_b200 import kitti_eval as K
from tests.test_kitti_eval import KEYS

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "eval_bootstrap.npz")
RANGES_GOLD = os.path.join(HERE, "golden", "eval_ranges.npz")
TABLES = (11, 40, "coco")
AP_KEYS = ("bbox", "bev", "d3", "aos")


def _frames():
    g = np.load(RANGES_GOLD)
    n = int(g["nframes"])
    gts = [{k: g["gt%d_%s" % (i, k)] for k in KEYS} for i in range(n)]
    dts = [{k: g["dt%d_%s" % (i, k)] for k in KEYS + ("score",)} for i in range(n)]
    return gts, dts


def _same(a, b, what=""):
    """Two (bootstrap) AP dicts equal bit for bit, NaN where NaN."""
    for k in AP_KEYS:
        if a[k] is None or b[k] is None:
            assert a[k] is None and b[k] is None, (what, k)
        else:
            x, y = np.asarray(a[k]), np.asarray(b[k])
            assert x.shape == y.shape and x.tobytes() == y.tobytes(), (what, k)


def _same_boot(a, b):
    assert a["bootstrap"].keys() == b["bootstrap"].keys()
    for t in a["bootstrap"]:
        _same(a["bootstrap"][t], b["bootstrap"][t], t)
    assert ("bootstrap_ranges" in a) == ("bootstrap_ranges" in b)
    for (lo, hi, x), (lo2, hi2, y) in zip(a.get("bootstrap_ranges", []), b.get("bootstrap_ranges", [])):
        assert (lo, hi) == (lo2, hi2)
        for t in x:
            _same(x[t], y[t], (lo, t))


# ------------------------------------------------------------------------------------------------------------ CPU
def test_host_path_equals_the_reference_per_replicate():
    gts, dts = _frames()
    g = np.load(GOLD)
    idx = g["idx"]
    ev = K.eval_many(gts, [dts], [0, 1, 2], (11, "coco"), O.rotate_iou_eval, bootstrap=idx)[0]["bootstrap"]
    assert ev[11]["d3"].shape == (len(idx), 3, 3, 2) and ev["coco"]["d3"].shape == (len(idx), 3, 3)
    for r in range(len(idx)):
        for tag, t in (("", 11), ("coco_", "coco")):
            for key in AP_KEYS:
                name = "r%d_%s%s" % (r, tag, key)
                if name in g.files:
                    assert ev[t][key][r].tobytes() == g[name].tobytes(), name
                else:
                    assert key == "aos" and not g["aos"][r] and np.isnan(ev[t][key][r]).all()
    assert g["aos"].any()
    # the draw without Pedestrian GT: AP 0 there
    assert not ev[11]["d3"][-1, 1].any() and ev[11]["d3"][-1, 0].any()


def test_identity_row_is_the_evaluation():
    gts, dts = _frames()
    sets = [dts, [dict(d, score=np.clip(d["score"] - 0.1, 0, 1)) for d in dts]]
    idx = np.stack([np.arange(len(gts)), np.arange(len(gts))[::-1]])
    evs = K.eval_many(gts, sets, [0, 1, 2], TABLES, O.rotate_iou_eval, ranges=[0, 20, np.inf], bootstrap=idx)
    for ev in evs:
        for t in TABLES:
            _same({k: None if v is None else v[0] for k, v in ev["bootstrap"][t].items()}, ev[t][1], t)
        for (_, _, full), (_, _, boot) in zip(ev["ranges"], ev["bootstrap_ranges"]):
            for t in TABLES:
                _same({k: None if v is None else v[0] for k, v in boot[t].items()}, full[t][1], t)


def test_a_set_against_itself_differs_by_nothing():
    gts, dts = _frames()
    idx = K.bootstrap_indices(len(gts), 4, seed=3)
    a, b = K.eval_many(gts, [dts, copy.deepcopy(dts)], [0, 1], (11,), O.rotate_iou_eval, bootstrap=idx)
    for key in ("bbox", "bev", "d3"):
        d = b["bootstrap"][11][key] - a["bootstrap"][11][key]
        assert not d.any()
        s = K.paired_summary(b["bootstrap"][11][key], a["bootstrap"][11][key])
        assert not s["interval"].any() and not s["better"].any()


def test_bootstrap_indices_rows_do_not_depend_on_r():
    a = K.bootstrap_indices(37, 5, seed=4)
    assert a.dtype == np.int64 and a.shape == (5, 37) and a.min() >= 0 and a.max() < 37
    np.testing.assert_array_equal(a, K.bootstrap_indices(37, 5, seed=4))
    np.testing.assert_array_equal(a[:2], K.bootstrap_indices(37, 2, seed=4))
    rs = np.random.RandomState(4)
    np.testing.assert_array_equal(a[0], rs.randint(0, 37, 37))
    np.testing.assert_array_equal(a[1], rs.randint(0, 37, 37))
    assert (a != K.bootstrap_indices(37, 5, seed=5)).any()


@pytest.mark.parametrize("bad", [np.zeros((2, 3), np.float64), np.zeros((0, 5), np.int64), np.zeros(5, np.int64),
                                 np.zeros((2, 4), np.int64), np.full((1, 5), 5), np.full((1, 5), -1),
                                 np.zeros((1, 5), bool), [[0, 1, 2, 3, "a"]]])
def test_bad_indices_are_refused(bad):
    gts, dts = _frames()
    with pytest.raises(ValueError, match="bootstrap"):
        K.eval_many(gts[:5], [dts[:5]], [0], (11,), O.rotate_iou_eval, bootstrap=bad)


def _kitti_args(root, extra):
    return ["--data-root", root, "--results", root] + extra


@pytest.mark.parametrize("extra, msg", [(["--bootstrap", "0"], "--bootstrap"), (["--bootstrap", "-3"], "--bootstrap"),
                                        (["--bootstrap-seed", "1"], "--bootstrap-seed")])
def test_bad_options_are_refused(extra, msg, tmp_path, capsys):
    from sassd_b200 import test as T
    root = str(tmp_path)
    os.makedirs(os.path.join(root, "ImageSets"))
    os.makedirs(os.path.join(root, "training", "label_2"))
    open(os.path.join(root, "ImageSets", "val.txt"), "w").close()
    with pytest.raises(SystemExit) as e:
        K.parse_args(_kitti_args(root, extra))
    assert e.value.code == 2 and msg in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        T.parse_args(["c.py", "a.pth", "--data-root", root] + extra)
    assert e.value.code == 2 and msg in capsys.readouterr().err
    for unlabelled in (["--split", "test", "--out", "o"], ["--drive", "d", "--out", "o"]):
        src = [] if unlabelled[0] == "--drive" else ["--data-root", root]
        with pytest.raises(SystemExit) as e:
            T.parse_args(["c.py", "a.pth"] + src + unlabelled + ["--bootstrap", "10"])
        assert e.value.code == 2 and "--bootstrap needs a labelled split" in capsys.readouterr().err


def test_command_arguments():
    from sassd_b200 import test as T
    a = T.parse_args(["c.py", "a.pth", "--data-root", "r", "--bootstrap", "100"])
    assert a.bootstrap == 100 and a.bootstrap_seed == 0
    a = T.parse_args(["c.py", "a.pth", "--data-root", "r", "--bootstrap", "5", "--bootstrap-seed", "9"])
    assert a.bootstrap_seed == 9
    a = T.parse_args(["c.py", "a.pth", "--data-root", "r"])
    assert a.bootstrap is None and a.bootstrap_seed is None and K.bootstrap_kw(a, 10) == {}


def test_helpers_are_numpy():
    rng = np.random.default_rng(0)
    a, b = rng.uniform(0, 100, (50, 3, 3)), rng.uniform(0, 100, (50, 3, 3))
    np.testing.assert_array_equal(K.percentile_interval(a), np.percentile(a, [2.5, 97.5], axis=0))
    s = K.paired_summary(a, b)
    np.testing.assert_array_equal(s["interval"], np.percentile(a - b, [2.5, 97.5], axis=0))
    np.testing.assert_array_equal(s["better"], np.mean(a - b > 0, axis=0))


def test_replicate_axis_tail_equals_per_replicate_tail():
    """_pr_arrays and _ap_dicts on [R, ...] arrays give each replicate what they give on its own arrays."""
    rng = np.random.default_rng(1)
    R, Kn, C, D, M = 5, 2, 3, 6, 12
    pr = rng.integers(0, 20, (R, Kn, C, D, 3, M, 41, 4)).astype(np.float64)
    pr[..., 3] = rng.uniform(0, 10, pr.shape[:-1])
    n_thresh = rng.integers(0, 42, (R, Kn, C, D, 3, M))
    flags = rng.uniform(size=(R, Kn)) < 0.5
    whole = K._pr_arrays(pr, n_thresh, flags)
    for r in range(R):
        one = K._pr_arrays(pr[r], n_thresh[r], flags[r])
        for k in range(Kn):
            for e0 in (0, 3):
                a = K._ap_dicts([p[k] for p in whole], e0, 3, TABLES, 2, True)
                b = K._ap_dicts([p[k] for p in one], e0, 3, TABLES, 2, True)
                for t in TABLES:
                    _same({x: a[t][x][r] for x in AP_KEYS}, b[t], (r, k, e0, t))


# ------------------------------------------------------------------------------------------------------------ GPU
def _device_overlaps(boxes, query, criterion):
    return K.rotate_iou_gpu_eval(boxes, query, criterion)


def _nan_sets(nsets):
    """The range test's edge sets (NaN locations) with NaN scores on a few detections of each set."""
    from tests.test_kitti_eval_ranges import _edge_sets
    gts, sets, edges = _edge_sets(nsets)
    for k, s in enumerate(sets):
        for f in (3 + k, 10, len(s) - 2):
            if len(s[f]["score"]):
                s[f] = dict(s[f], score=s[f]["score"].copy())
                s[f]["score"][0] = np.nan
    return gts, sets, edges


@pytest.mark.gpu
@pytest.mark.parametrize("nsets", [1, 3])
def test_device_equals_host_bit_for_bit(nsets, monkeypatch):
    monkeypatch.setattr(K, "BOOTSTRAP_CHUNK", 3)
    gts, sets, edges = _nan_sets(nsets)
    idx = K.bootstrap_indices(len(gts), 7, seed=nsets)
    idx[0] = np.arange(len(gts))
    idx[1] = 4
    for ranges in (None, edges):
        dev = K.eval_many(gts, sets, [0, 1, 2], TABLES, ranges=ranges, bootstrap=idx)
        host = K.eval_many(gts, sets, [0, 1, 2], TABLES, _device_overlaps, ranges=ranges, bootstrap=idx)
        plain = K.eval_many(gts, sets, [0, 1, 2], TABLES, ranges=ranges)
        for a, b, p in zip(dev, host, plain):
            _same_boot(a, b)
            for t in TABLES:          # the evaluation itself is unchanged by the bootstrap
                assert a[t][0] == p[t][0]
                _same(a[t][1], p[t][1], t)
                _same({x: None if v is None else v[0] for x, v in a["bootstrap"][t].items()}, p[t][1], t)


@pytest.mark.gpu
def test_device_equals_the_reference_goldens():
    gts, dts = _frames()
    g = np.load(GOLD)
    ev = K.eval_many(gts, [dts], [0, 1, 2], (11, "coco"), bootstrap=g["idx"])[0]["bootstrap"]
    for r in range(len(g["idx"])):
        for tag, t in (("", 11), ("coco_", "coco")):
            for key in AP_KEYS:
                name = "r%d_%s%s" % (r, tag, key)
                if name in g.files:
                    assert ev[t][key][r].tobytes() == g[name].tobytes(), name


@pytest.mark.gpu
def test_every_replicate_of_a_full_split_is_its_evaluation():
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden_eval import synth_annos
    gts, dts = synth_annos(np.random.default_rng(21), 3769)
    sets = [dts, [dict(d, score=np.clip(d["score"] + 0.05 * np.sin(np.arange(len(d["score"]))), 0, 1)) for d in dts]]
    idx = K.bootstrap_indices(len(gts), 16, seed=2)
    evs = K.eval_many(gts, sets, ["Car", "Pedestrian", "Cyclist"], (11, "coco"), bootstrap=idx)
    for r in range(len(idx)):
        one = K.eval_many([gts[i] for i in idx[r]], [[d[i] for i in idx[r]] for d in sets],
                          ["Car", "Pedestrian", "Cyclist"], (11, "coco"))
        for ev, o in zip(evs, one):
            for t in (11, "coco"):
                _same({x: None if v is None else v[r] for x, v in ev["bootstrap"][t].items()}, o[t][1], (r, t))


@pytest.mark.gpu
def test_eval_command_with_bootstrap(tmp_path):
    from sassd_b200 import kitti_data as KD
    from sassd_b200 import test as T
    from tests.kitti_root import write_tree
    from tests.test_kitti_eval_coco import _perturbed_sets
    root = str(tmp_path / "kitti")
    write_tree(root)
    ids = KD.read_split(root, "trainval")
    gt = KD.read_labels(os.path.join(root, "training", "label_2"), ids)
    sets = _perturbed_sets([dict({k: g[k] for k in KEYS}, score=np.linspace(0.2, 0.9, len(g["name"]))) for g in gt], 2,
                           seed=9)
    dirs = []
    for k, s in enumerate(sets):
        dirs.append(str(tmp_path / ("set%d" % k)))
        T.write_results(dirs[-1], ids, [dict(a, dimensions=np.asarray(a["dimensions"], np.float64)) for a in s])
    base = ["--data-root", root, "--split", "trainval", "--results"] + dirs + ["--classes", "Car", "Pedestrian",
                                                                                "--r40", "--coco"]
    js = str(tmp_path / "e.json")
    printed = []
    res = K.main(base + ["--bootstrap", "20", "--bootstrap-seed", "3", "--json", js],
                 log=lambda *a, **k: printed.append(" ".join(str(x) for x in a)))
    plain = K.main(base, log=lambda *a, **k: None)
    for e, p in zip(res["results"], plain["results"]):
        assert all(e[k] == p[k] for k in p if k != "times_s")
        assert set(e) == set(p)
    boot = res["bootstrap"]
    assert (boot["replicates"], boot["seed"], boot["frames"]) == (20, 3, len(ids))
    want = K.eval_many(KD.read_labels(os.path.join(root, "training", "label_2"), ids),
                       [KD.read_labels(d, ids) for d in dirs], ["Car", "Pedestrian"], (11, 40, "coco"),
                       bootstrap=K.bootstrap_indices(len(ids), 20, 3))
    for s, w in zip(boot["sets"], want):
        assert s["intervals"]["11"]["d3"] == K.percentile_interval(w["bootstrap"][11]["d3"]).tolist()
        assert s["intervals"]["coco"]["bev"] == K.percentile_interval(w["bootstrap"]["coco"]["bev"]).tolist()
    pair = K.paired_summary(want[1]["bootstrap"][11]["d3"][:, 0, 1, 0], want[0]["bootstrap"][11]["d3"][:, 0, 1, 0])
    got = [p for p in boot["paired"] if p["table"] == "11" and p["cls"] == "Car"]
    assert got[0]["interval"] == pair["interval"].tolist() and got[0]["better"] == float(pair["better"])
    assert any(p.startswith("paired against %s" % dirs[0]) for p in printed)
    assert any(p.startswith("Car AP 95% interval (20 replicates):") for p in printed)
    line = printed[printed.index("summary: 2 directories (moderate 3D AP)") + 1]
    assert "Car 3d mod 95% R11 [" in line and " COCO [" in line
    with open(js) as fh:
        assert json.dumps(json.load(fh)["bootstrap"]) == json.dumps(boot)      # NaN (no AOS) != NaN: compare texts


@pytest.mark.gpu
def test_driver_bootstrap_for_a_sweep_equals_single_runs(tmp_path):
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
            "--coco"]
    boot = ["--bootstrap", "12", "--bootstrap-seed", "5"]
    singles = []
    for c in ckpts:
        res = T.run(T.parse_args([CAR_CFG, c] + base + boot), log=lambda *a, **k: None)
        plain = T.run(T.parse_args([CAR_CFG, c] + base), log=lambda *a, **k: None)
        for key in ("text", "ap", "text_coco", "ap_coco"):
            assert res[key] == plain[key], key
        singles.append(res)
    printed = []
    res = T.run(T.parse_args([CAR_CFG, ckpts[0], "--checkpoints", ckpts[1]] + base + boot),
                log=lambda *a, **k: printed.append(" ".join(str(x) for x in a)))
    for k, (e, single) in enumerate(zip(res["checkpoints"], singles)):
        for key in ("text", "ap", "text_coco", "ap_coco"):
            assert e[key] == single[key], key
        assert res["bootstrap"]["sets"][k]["intervals"] == single["bootstrap"]["sets"][0]["intervals"]
    assert len(res["bootstrap"]["paired"]) == 2          # R11 and COCO, Car
    assert any(p.startswith("paired against %s" % os.path.basename(ckpts[0])) for p in printed)

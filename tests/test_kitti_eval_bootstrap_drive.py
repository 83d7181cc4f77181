"""Drive-level bootstrap replicates and per-drive AP (kitti_eval.ReplicateLists, bootstrap_groups, per_drive_report,
kitti_data.read_drive_mapping / split_drives, --bootstrap-by / --mapping / --per-drive of both commands).

* CPU: the devkit mapping reader and its refusals; bootstrap_groups' rows (deterministic, independent of R, each drawn
  drive's frames ascending, bootstrap_indices' rows for one frame per drive); ReplicateLists' refusals; the host path
  (the oracle's rotated overlaps injected) equals the unmodified reference on each list of
  tests/golden/eval_bootstrap_drive.npz (make_golden_eval_bootstrap_drive.py: grouped draws, one drive drawn G times,
  a one-frame list, a list whose first frame has no detections); the options of both commands.
* GPU: the device path equals the host path and the reference bit for bit on lists of any length; the array form and
  the same rows as ReplicateLists give the same bits; every drive-level replicate of 3769 synthetic frames equals
  eval_many on its list; both commands with --bootstrap-by drive --per-drive keep their tables, give a sweep's
  checkpoints their single runs' intervals, and print each drive's own evaluation.
"""
import json
import os

import numpy as np
import pytest

from oracle import kitti_eval as O
from sassd_b200 import kitti_data as KD
from sassd_b200 import kitti_eval as K
from tests.test_kitti_eval import KEYS
from tests.test_kitti_eval_bootstrap import AP_KEYS, TABLES, _frames, _same, _same_boot

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "eval_bootstrap_drive.npz")


def write_mapping(mapping_dir, drives, seed=0):
    """The devkit's mapping files for training frames whose drives are ``drives`` (one name per frame id): the mapping
    lines in a shuffled order, train_rand pointing each frame at its line."""
    os.makedirs(mapping_dir, exist_ok=True)
    order = np.random.RandomState(seed).permutation(len(drives))      # line j holds frame order[j]
    with open(os.path.join(mapping_dir, "train_mapping.txt"), "w") as fh:
        for f in order:
            fh.write("%s %s %010d\n" % (drives[f][:10], drives[f], f))
    line_of = np.empty(len(drives), np.int64)
    line_of[order] = np.arange(1, len(drives) + 1)
    with open(os.path.join(mapping_dir, "train_rand.txt"), "w") as fh:
        fh.write(",".join(str(int(l)) for l in line_of) + "\n")


def _drive_names(n, sizes):
    """n frames in consecutive runs of ``sizes`` (the last run takes the rest), named as KITTI raw drives."""
    names, d = [], 0
    while len(names) < n:
        names += ["2011_09_26_drive_%04d_sync" % (d + 1)] * sizes[d % len(sizes)]
        d += 1
    return names[:n]


def _gold_frames():
    """The golden's frames: eval_ranges.npz's plus frame ``empty_of``'s GT without detections."""
    g = np.load(GOLD)
    gts, dts = _frames()
    e = int(g["empty_of"])
    gts.append(gts[e])
    dts.append({k: v[:0] for k, v in dts[e].items()})
    return gts, dts, g


def _gold_lists(g):
    return K.ReplicateLists([g["flat"][g["off"][r]:g["off"][r + 1]] for r in range(len(g["off"]) - 1)])


def _row(ap, r):
    return {k: None if v is None else v[r] for k, v in ap.items()}


# ------------------------------------------------------------------------------------------------------------ CPU
def test_read_drive_mapping(tmp_path):
    drives = _drive_names(23, [5, 1, 9])
    write_mapping(str(tmp_path), drives, seed=3)
    assert KD.read_drive_mapping(str(tmp_path)) == drives
    got = KD.split_drives(drives, [4, 0, 22, 5])
    assert got.tolist() == [drives[4], drives[0], drives[22], drives[5]]
    with pytest.raises(ValueError, match="frame 000023"):
        KD.split_drives(drives, [1, 23])


@pytest.mark.parametrize("case, msg", [
    ("fields", r"train_mapping\.txt line 2"), ("not_int", r"train_rand\.txt entry 1"),
    ("range", r"train_rand\.txt entry 3"), ("zero", r"train_rand\.txt entry 0"),
    ("twice", r"train_rand\.txt entry 4"), ("short", r"train_rand\.txt has 4 entries")])
def test_read_drive_mapping_refusals(case, msg, tmp_path):
    d = str(tmp_path)
    write_mapping(d, _drive_names(5, [2]))
    lines = open(os.path.join(d, "train_mapping.txt")).read().splitlines()
    rand = ["1", "2", "3", "4", "5"]
    if case == "fields":
        lines[1] = "2011_09_26 2011_09_26_drive_0001_sync"
    elif case == "not_int":
        rand[1] = "x"
    elif case == "range":
        rand[3] = "6"
    elif case == "zero":
        rand[0] = "0"
    elif case == "twice":
        rand[4] = "2"
    else:
        rand = rand[:4]
    with open(os.path.join(d, "train_mapping.txt"), "w") as fh:
        fh.write("\n".join(lines) + "\n")
    with open(os.path.join(d, "train_rand.txt"), "w") as fh:
        fh.write(",".join(rand) + "\n")
    with pytest.raises(ValueError, match=msg):
        KD.read_drive_mapping(d)


def test_bootstrap_groups_rows():
    groups = np.array(["b", "a", "c", "a", "b", "b", "d"])
    lists = K.bootstrap_groups(groups, 6, seed=4)
    assert len(lists) == 6 and lists.flat.dtype == np.int64 and lists.off.dtype == np.int64
    members = {"a": [1, 3], "b": [0, 4, 5], "c": [2], "d": [6]}
    rs = np.random.RandomState(4)
    for r in range(6):
        draw = rs.randint(0, 4, 4)
        want = np.concatenate([members["abcd"[g]] for g in draw])
        np.testing.assert_array_equal(lists[r], want)
    again = K.bootstrap_groups(groups, 2, seed=4)
    np.testing.assert_array_equal(again.flat, lists.flat[:again.off[-1]])
    np.testing.assert_array_equal(again.off, lists.off[:3])
    assert not np.array_equal(K.bootstrap_groups(groups, 6, seed=5).flat, lists.flat)


def test_one_frame_per_group_is_bootstrap_indices():
    for F in (1, 7, 40):
        idx = K.bootstrap_indices(F, 9, seed=F)
        lists = K.bootstrap_groups(np.arange(F), 9, seed=F)
        np.testing.assert_array_equal(lists.off, np.arange(10) * F)
        for r in range(9):
            np.testing.assert_array_equal(lists[r], idx[r])


def test_golden_grouped_draws_are_bootstrap_groups():
    g = np.load(GOLD)
    n = int(g["ordinary"])
    lists = K.bootstrap_groups(g["groups"], n, seed=7)
    np.testing.assert_array_equal(lists.flat, g["flat"][:g["off"][n]])
    np.testing.assert_array_equal(lists.off, g["off"][:n + 1])


@pytest.mark.parametrize("bad", [[], [np.array([], np.int64)], [np.array([0, 1]), np.array([], np.int64)],
                                 [np.array([0.0, 1.0])], [np.array([[0, 1]])], [np.array([True, False])],
                                 [np.array(["0"])]])
def test_bad_replicate_lists_are_refused(bad):
    with pytest.raises(ValueError, match="bootstrap"):
        K.ReplicateLists(bad)


@pytest.mark.parametrize("row", [[0, 5], [-1, 2], [4, 4, 4, 4, 4, 4, 4, 4, 9]])
def test_replicate_lists_outside_the_frames_are_refused(row):
    gts, dts = _frames()
    with pytest.raises(ValueError, match="bootstrap"):
        K.eval_many(gts[:5], [dts[:5]], [0], (11,), O.rotate_iou_eval,
                    bootstrap=K.ReplicateLists([np.array([0, 1]), np.array(row)]))


def test_host_path_equals_the_reference_per_list():
    gts, dts, g = _gold_frames()
    lists = _gold_lists(g)
    assert len(set(lists.lengths.tolist())) > 2 and 1 in lists.lengths and lists.lengths.max() > len(gts)
    assert not len(dts[lists[len(lists) - 1][0]]["name"])
    ev = K.eval_many(gts, [dts], [0, 1, 2], (11, "coco"), O.rotate_iou_eval, bootstrap=lists)[0]["bootstrap"]
    for r in range(len(lists)):
        for tag, t in (("", 11), ("coco_", "coco")):
            for key in AP_KEYS:
                name = "r%d_%s%s" % (r, tag, key)
                if name in g.files:
                    assert ev[t][key][r].tobytes() == g[name].tobytes(), name
                else:
                    assert key == "aos" and not g["aos"][r] and np.isnan(ev[t][key][r]).all()


def _kitti_root(tmp_path):
    root = str(tmp_path)
    os.makedirs(os.path.join(root, "ImageSets"))
    os.makedirs(os.path.join(root, "training", "label_2"))
    open(os.path.join(root, "ImageSets", "val.txt"), "w").close()
    return root


@pytest.mark.parametrize("extra, msg", [
    (["--bootstrap-by", "drive", "--mapping", "m"], "--bootstrap-by goes with --bootstrap"),
    (["--bootstrap-by", "frame"], "--bootstrap-by goes with --bootstrap"),
    (["--bootstrap", "5", "--bootstrap-by", "drive"], "--bootstrap-by drive needs --mapping"),
    (["--per-drive"], "--per-drive needs --mapping"),
    (["--mapping", "m"], "--mapping goes with"),
    (["--bootstrap", "5", "--mapping", "m"], "--mapping goes with"),
    (["--bootstrap", "5", "--bootstrap-by", "frame", "--mapping", "m"], "--mapping goes with"),
    (["--bootstrap", "5", "--bootstrap-by", "block"], "--bootstrap-by")])
def test_bad_options_are_refused(extra, msg, tmp_path, capsys):
    from sassd_b200 import test as T
    root = _kitti_root(tmp_path)
    with pytest.raises(SystemExit) as e:
        K.parse_args(["--data-root", root, "--results", root] + extra)
    assert e.value.code == 2 and msg in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        T.parse_args(["c.py", "a.pth", "--data-root", root] + extra)
    assert e.value.code == 2 and msg in capsys.readouterr().err


@pytest.mark.parametrize("extra, flag", [
    (["--bootstrap", "5", "--bootstrap-by", "drive", "--mapping", "m"], "--bootstrap"),
    (["--per-drive", "--mapping", "m"], "--mapping"), (["--mapping", "m"], "--mapping"),
    (["--per-drive"], "--per-drive"), (["--bootstrap-by", "frame"], "--bootstrap-by")])
def test_unlabelled_sources_refuse_the_options(extra, flag, tmp_path, capsys):
    from sassd_b200 import test as T
    root = _kitti_root(tmp_path)
    for unlabelled in (["--data-root", root, "--split", "test", "--out", "o"], ["--drive", "d", "--out", "o"]):
        with pytest.raises(SystemExit) as e:
            T.parse_args(["c.py", "a.pth"] + unlabelled + extra)
        assert e.value.code == 2 and "%s needs a labelled split" % flag in capsys.readouterr().err


def test_command_arguments(tmp_path):
    from sassd_b200 import test as T
    root = _kitti_root(tmp_path)
    a = T.parse_args(["c.py", "a.pth", "--data-root", root, "--bootstrap", "10"])
    assert a.bootstrap_by == "frame" and a.mapping is None and not a.per_drive
    a = K.parse_args(["--data-root", root, "--results", root, "--bootstrap", "10", "--bootstrap-by", "drive",
                      "--mapping", "m", "--per-drive"])
    assert (a.bootstrap, a.bootstrap_by, a.mapping, a.per_drive) == (10, "drive", "m", True)
    a = T.parse_args(["c.py", "a.pth", "--data-root", root, "--mapping", "m", "--per-drive"])
    assert a.bootstrap is None and a.bootstrap_by is None and K.bootstrap_kw(a, 10) == {}
    drives = np.array(["x", "y", "x", "z"])
    a = K.parse_args(["--data-root", root, "--results", root, "--bootstrap", "4", "--bootstrap-seed", "2",
                      "--bootstrap-by", "drive", "--mapping", "m"])
    kw = K.bootstrap_kw(a, 4, drives)
    want = K.bootstrap_groups(drives, 4, 2)
    assert np.array_equal(kw["bootstrap"].flat, want.flat) and np.array_equal(kw["bootstrap"].off, want.off)
    assert K.bootstrap_groups_of(a, drives) == 3


# ------------------------------------------------------------------------------------------------------------ GPU
def _device_overlaps(boxes, query, criterion):
    return K.rotate_iou_gpu_eval(boxes, query, criterion)


@pytest.mark.gpu
@pytest.mark.parametrize("nsets", [1, 3])
def test_device_equals_host_on_lists_of_any_length(nsets, monkeypatch):
    from tests.test_kitti_eval_bootstrap import _nan_sets
    monkeypatch.setattr(K, "BOOTSTRAP_CHUNK", 3)
    gts, sets, edges = _nan_sets(nsets)
    F = len(gts)
    groups = np.random.RandomState(nsets).randint(0, 6, F)
    drawn = K.bootstrap_groups(groups, 5, seed=nsets)
    rows = list(drawn) + [np.arange(F), np.tile(np.flatnonzero(groups == groups[0]), 6), np.array([F - 1]),
                          np.arange(F)[::-1][:F // 3]]
    lists = K.ReplicateLists(rows)
    for ranges in (None, edges):
        dev = K.eval_many(gts, sets, [0, 1, 2], TABLES, ranges=ranges, bootstrap=lists)
        host = K.eval_many(gts, sets, [0, 1, 2], TABLES, _device_overlaps, ranges=ranges, bootstrap=lists)
        plain = K.eval_many(gts, sets, [0, 1, 2], TABLES, ranges=ranges)
        for a, b, p in zip(dev, host, plain):
            _same_boot(a, b)
            for t in TABLES:
                assert a[t][0] == p[t][0]
                _same(_row(a["bootstrap"][t], 5), p[t][1], t)          # the identity list


@pytest.mark.gpu
def test_device_equals_the_reference_goldens():
    gts, dts, g = _gold_frames()
    ev = K.eval_many(gts, [dts], [0, 1, 2], (11, "coco"), bootstrap=_gold_lists(g))[0]["bootstrap"]
    for r in range(len(g["off"]) - 1):
        for tag, t in (("", 11), ("coco_", "coco")):
            for key in AP_KEYS:
                name = "r%d_%s%s" % (r, tag, key)
                if name in g.files:
                    assert ev[t][key][r].tobytes() == g[name].tobytes(), name
                else:
                    assert np.isnan(ev[t][key][r]).all(), name


@pytest.mark.gpu
def test_array_and_replicate_lists_give_the_same_bits(monkeypatch):
    from tests.test_kitti_eval_bootstrap import _nan_sets
    monkeypatch.setattr(K, "BOOTSTRAP_CHUNK", 4)
    gts, sets, edges = _nan_sets(3)
    idx = K.bootstrap_indices(len(gts), 9, seed=11)
    a = K.eval_many(gts, sets, [0, 1, 2], TABLES, ranges=edges, bootstrap=idx)
    b = K.eval_many(gts, sets, [0, 1, 2], TABLES, ranges=edges, bootstrap=K.ReplicateLists(list(idx)))
    for x, y in zip(a, b):
        _same_boot(x, y)


@pytest.mark.gpu
def test_every_drive_level_replicate_of_a_full_split_is_its_evaluation(tmp_path):
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden_eval import synth_annos
    gts, dts = synth_annos(np.random.default_rng(21), 3769)
    sets = [dts, [dict(d, score=np.clip(d["score"] + 0.05 * np.sin(np.arange(len(d["score"]))), 0, 1)) for d in dts]]
    ids = np.arange(3769)
    write_mapping(str(tmp_path), _drive_names(7481, [37, 112, 64, 230, 18, 95]), seed=1)
    drives = KD.split_drives(KD.read_drive_mapping(str(tmp_path)), ids)
    lists = K.bootstrap_groups(drives, 8, seed=2)
    assert len(set(lists.lengths.tolist())) > 1
    evs = K.eval_many(gts, sets, ["Car", "Pedestrian", "Cyclist"], (11, "coco"), bootstrap=lists)
    for r in range(len(lists)):
        one = K.eval_many([gts[i] for i in lists[r]], [[d[i] for i in lists[r]] for d in sets],
                          ["Car", "Pedestrian", "Cyclist"], (11, "coco"))
        for ev, o in zip(evs, one):
            for t in (11, "coco"):
                _same(_row(ev["bootstrap"][t], r), o[t][1], (r, t))


ROOT_DRIVES = ["2011_09_26_drive_0001_sync"] * 3 + ["2011_09_28_drive_0002_sync"] * 2 + \
              ["2011_10_03_drive_0003_sync"] * 3          # training frames 0..7 of tests/kitti_root.py


def _same_ap_lists(got, ap):
    """A per-drive JSON AP dict against an eval_many AP dict: bbox / BEV / 3D equal, AOS where the drive has it."""
    for k in ("bbox", "bev", "d3"):
        assert got[k] == np.asarray(ap[k]).tolist(), k
    if ap["aos"] is not None:
        assert got["aos"] == np.asarray(ap["aos"]).tolist()


def _check_per_drive(per_drive, gt, sets, classes, tables):
    drives = np.array(ROOT_DRIVES)[[0, 1, 2, 3, 4, 6, 5, 7]]
    assert [d["drive"] for d in per_drive] == sorted(set(ROOT_DRIVES))
    for d in per_drive:
        rows = np.flatnonzero(drives == d["drive"])
        assert d["frames"] == len(rows)
        one = K.eval_many([gt[i] for i in rows], [[s[i] for i in rows] for s in sets], classes, tables)
        for col, o in zip(d["sets"], one):
            for t in tables:
                _same_ap_lists(col["ap"][str(t)], o[t][1])


@pytest.mark.gpu
def test_eval_command_drive_level_and_per_drive(tmp_path):
    from sassd_b200 import test as T
    from tests.kitti_root import write_tree
    from tests.test_kitti_eval_coco import _perturbed_sets
    root = str(tmp_path / "kitti")
    write_tree(root)
    mapping = os.path.join(root, "mapping")
    write_mapping(mapping, ROOT_DRIVES, seed=2)
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
    boot = ["--bootstrap", "30", "--bootstrap-seed", "3"]
    js = str(tmp_path / "e.json")
    printed, frame_printed, plain_printed = [], [], []
    res = K.main(base + boot + ["--bootstrap-by", "drive", "--mapping", mapping, "--per-drive", "--json", js],
                 log=lambda *a, **k: printed.append(" ".join(str(x) for x in a)))
    frame = K.main(base + boot, log=lambda *a, **k: frame_printed.append(" ".join(str(x) for x in a)))
    plain = K.main(base, log=lambda *a, **k: plain_printed.append(" ".join(str(x) for x in a)))
    for e, f, p in zip(res["results"], frame["results"], plain["results"]):
        assert all(e[k] == p[k] for k in p) and set(e) == set(f)
    # the frame-level run is what it was: its blocks and JSON entry
    assert sorted(frame["bootstrap"]) == ["frames", "paired", "replicates", "seed", "sets"]
    assert "per_drive" not in frame and any(l.startswith("Car AP 95% interval (30 replicates):") for l in frame_printed)
    assert not any("drive-level" in l or l.startswith("per drive") for l in frame_printed + plain_printed)
    want = K.eval_many(gt, [KD.read_labels(d, ids) for d in dirs], ["Car", "Pedestrian"], (11, 40, "coco"),
                       bootstrap=K.bootstrap_groups(np.array(ROOT_DRIVES)[ids], 30, 3))
    b = res["bootstrap"]
    assert (b["by"], b["groups"], b["replicates"], b["seed"], b["frames"]) == ("drive", 3, 30, 3, len(ids))
    lengths = K.bootstrap_groups(np.array(ROOT_DRIVES)[ids], 30, 3).lengths
    assert b["lengths"] == dict(min=int(lengths.min()), median=float(np.median(lengths)), max=int(lengths.max()))
    for s, w in zip(b["sets"], want):
        assert s["intervals"]["11"]["d3"] == K.percentile_interval(w["bootstrap"][11]["d3"]).tolist()
        assert s["intervals"]["coco"]["bev"] == K.percentile_interval(w["bootstrap"]["coco"]["bev"]).tolist()
    assert any(l.startswith("Car AP 95% interval (30 drive-level replicates of 3 drives):") for l in printed)
    assert any(l.startswith("paired against %s (moderate 3D AP, 30 drive-level replicates of 3 drives):" % dirs[0])
               for l in printed)
    head = printed.index("per drive (moderate 3D AP, 3 drives; columns: %s):" % " | ".join(dirs))
    for line, name in zip(printed[head + 1:head + 4], sorted(set(ROOT_DRIVES))):
        assert line.startswith(name) and line.count("|") == 1 and " R40 " in line and " COCO " in line
    _check_per_drive(res["per_drive"], gt, [KD.read_labels(d, ids) for d in dirs], ["Car", "Pedestrian"],
                     (11, 40, "coco"))
    with open(js) as fh:
        assert json.dumps(json.load(fh)["per_drive"]) == json.dumps(res["per_drive"])


@pytest.mark.gpu
def test_driver_drive_level_sweep_equals_single_runs(tmp_path):
    from sassd_b200 import checkpoint
    from sassd_b200 import test as T
    from tests.checkpoint_weights import CAR_CFG, checkpoint_state_dict
    from tests.kitti_root import write_tree
    root = str(tmp_path / "kitti")
    write_tree(root)
    mapping = os.path.join(root, "mapping")
    write_mapping(mapping, ROOT_DRIVES, seed=4)
    ckpts = []
    for seed in (1, 2):
        ckpts.append(str(tmp_path / ("epoch_%d.pth" % seed)))
        checkpoint.save_checkpoint(checkpoint_state_dict(seed), ckpts[-1])
    base = ["--data-root", root, "--split", "trainval", "--lidar", "velodyne", "--batch", "4", "--workers", "2",
            "--coco"]
    opts = ["--bootstrap", "12", "--bootstrap-seed", "5", "--bootstrap-by", "drive", "--mapping", mapping,
            "--per-drive"]
    singles = []
    for c in ckpts:
        res = T.run(T.parse_args([CAR_CFG, c] + base + opts), log=lambda *a, **k: None)
        plain = T.run(T.parse_args([CAR_CFG, c] + base), log=lambda *a, **k: None)
        for key in ("text", "ap", "text_coco", "ap_coco"):
            assert res[key] == plain[key], key
        assert res["bootstrap"]["by"] == "drive" and res["bootstrap"]["groups"] == 3
        singles.append(res)
    # each drive's line is the evaluation of a run over that drive's frames alone
    for d in singles[0]["per_drive"]:
        frames = [i for i, name in enumerate(ROOT_DRIVES) if name == d["drive"]]
        with open(os.path.join(root, "ImageSets", d["drive"] + ".txt"), "w") as fh:
            fh.write("".join("%06d\n" % i for i in frames))
        one = T.run(T.parse_args([CAR_CFG, ckpts[0]] + base[:2] + ["--split", d["drive"]] + base[4:]),
                    log=lambda *a, **k: None)
        assert d["frames"] == len(frames)
        assert d["sets"][0]["ap"]["11"] == one["ap"] and d["sets"][0]["ap"]["coco"] == one["ap_coco"]
    printed = []
    res = T.run(T.parse_args([CAR_CFG, ckpts[0], "--checkpoints", ckpts[1]] + base + opts),
                log=lambda *a, **k: printed.append(" ".join(str(x) for x in a)))
    for k, (e, single) in enumerate(zip(res["checkpoints"], singles)):
        for key in ("text", "ap", "text_coco", "ap_coco"):
            assert e[key] == single[key], key
        assert res["bootstrap"]["sets"][k]["intervals"] == single["bootstrap"]["sets"][0]["intervals"]
        for d, ds in zip(res["per_drive"], single["per_drive"]):
            assert json.dumps(d["sets"][k]["ap"]) == json.dumps(ds["sets"][0]["ap"])
    assert res["bootstrap"]["lengths"] == singles[0]["bootstrap"]["lengths"]
    assert len(res["bootstrap"]["paired"]) == 2          # R11 and COCO, Car
    assert any(p.startswith("paired against %s (moderate 3D AP, 12 drive-level replicates of 3 drives):"
                            % os.path.basename(ckpts[0])) for p in printed)
    assert any(p.startswith("per drive (moderate 3D AP, 3 drives; columns: ") for p in printed)

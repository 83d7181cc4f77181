"""Road planes in the training-time augmentation (the reference's data.train.with_plane): kitti_data.read_plane,
augment.plane_shift, PointAugmentor.augment(road_planes=, calibs=), the assemble kernel's per-record height move and
the driver, against tests/golden/augment_plane.npz, produced by the reference's own get_road_plane, sample_all and
prepare_train_img steps with numba compiled (tests/golden/make_golden_augment_plane.py) on the synthetic root of
tests/kitti_root.py with tests/kitti_planes.py's plane files and overhang.

Bar: the plane, each sampled box's height move and moved box bit-equal to the reference's; every draw, sampled record,
noise index, final box and label, keep flag and augmented-cloud digest identical, at batch 1 and batch 4."""
import hashlib
import os
import pickle
import re
import shutil

import numpy as np
import pytest

from tests import kitti_planes as KP
from tests import kitti_root as KR
from tests.test_augment import CONFIGS, RUNS, _augmentor, _frame, _restore, _split, sha


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "augment_plane.npz"))


@pytest.fixture(scope="module")
def tree(tmp_path_factory, golden_dir):
    """The synthetic root with its plane files, the overhang, and the reference's kitti_dbinfos_train.pkl (the
    overhang's frame has no GT box, so the database is create_data.npz's)."""
    cd = np.load(os.path.join(golden_dir, "create_data.npz"))
    root = str(tmp_path_factory.mktemp("kitti_plane") / "kitti")
    KR.write_tree(root)
    KP.write_planes(root)
    KP.add_overhang(root)
    with open(os.path.join(root, "kitti_dbinfos_train.pkl"), "wb") as fh:
        pickle.dump(_restore(KR.unflatten(cd, "dbinfos_train")), fh)
    return root


def _plane_and_calib(root, idx):
    from sassd_b200.kitti_data import read_plane
    from sassd_b200.results import Calibration
    d = os.path.join(root, "training")
    return (read_plane(os.path.join(d, "planes", "%06d.txt" % idx)),
            Calibration(os.path.join(d, "calib", "%06d.txt" % idx)))


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


# ------------------------------------------------------------------ CPU
def test_read_plane_matches_the_reference(gold, tree):
    from sassd_b200.kitti_data import read_plane
    for f, idx in enumerate(KR.TRAIN):
        p = read_plane(os.path.join(tree, "training", "planes", "%06d.txt" % idx))
        assert p.dtype == np.float64 and p.shape == (4,)
        assert np.array_equal(_bits(p), _bits(gold["car_s0_plane"][f])), idx
        assert p[1] < 0, "the normal faces up"
    flipped = [i for i in KR.TRAIN if KP.PLANES[i][4]]
    assert flipped, "the fixture has planes written with b > 0"


@pytest.mark.parametrize("cfg,seed", RUNS)
def test_plane_shift_and_host_boxes_match_the_reference(gold, tree, cfg, seed):
    from sassd_b200.augment import plane_shift
    aug = _augmentor(tree, cfg, seed)
    key = "%s_s%d" % (cfg, seed)
    ns = gold[key + "_nsampled"]
    mvs, sampled = _split(gold, key, "mv", ns), _split(gold, key, "sampled", ns)
    sels = _split(gold, key, "sel", gold[key + "_nsel"])
    boxes = _split(gold, key, "boxes", gold[key + "_nbox"])
    labels = _split(gold, key, "labels", gold[key + "_nbox"])
    for f, idx in enumerate(KR.TRAIN):
        gt, names = _frame(tree, idx)
        plane, calib = _plane_and_calib(tree, idx)
        plan = aug.draw(gt, names, CONFIGS[cfg]["class_names"], plane, calib)
        assert ";".join(aug.records[r]["path"] for r in plan["records"]) == gold[key + "_paths"][f], (key, f)
        assert sha(plan["loc"]) == gold[key + "_loc_sha"][f] and sha(plan["rot"]) == gold[key + "_rot_sha"][f]
        assert (plan["flip"], plan["angle"], plan["scale"]) == (
            bool(gold[key + "_flip"][f]), gold[key + "_angle"][f], gold[key + "_scale"][f])
        assert len(plan["records"]) == ns[f] > 0
        assert np.array_equal(_bits(plan["mv"]), _bits(mvs[f])), (key, f)
        assert np.array_equal(_bits(plan["sampled"]), _bits(sampled[f])), (key, f)
        b64 = np.stack([aug.records[r]["box3d_lidar"] for r in plan["records"]])
        b32, mv = plane_shift(b64, plane, calib)
        assert np.array_equal(_bits(b32), _bits(sampled[f])) and np.array_equal(_bits(mv), _bits(mvs[f]))
        b, lab = aug.finish_boxes(plan, sels[f])
        assert np.array_equal(_bits(b), _bits(boxes[f])), (key, f)
        assert np.array_equal(lab, labels[f])
        assert (len(b) > 0) == bool(gold[key + "_keep"][f])
    f = KR.TRAIN.index(KP.OVERHANG_FRAME)
    assert gold[key + "_lift_crop"][f] > 0, "the lifted box crops overhang points the database box leaves"


def test_plane_shift_subtracts_the_move_rather_than_assigning_the_height():
    """z - (z - cur) is not always cur in float64: plane_shift keeps the reference's subtraction."""
    from sassd_b200.augment import plane_shift
    from sassd_b200.results import Calibration, project_rect_to_velo, project_velo_to_rect
    calib = Calibration(dict((k, v) for k, v in KR._rig(0).items() if k in ("P2", "Tr_velo_to_cam", "R0_rect")))
    rng = np.random.default_rng(3)
    b64 = np.concatenate([rng.uniform([5, -20, -0.5], [60, 20, 2.5], (4000, 3)),
                          np.tile([1.6, 3.9, 1.56, 0.3], (4000, 1))], 1)
    plane = np.array([-0.0106, -1.0, 0.0105, 1.658]) / np.linalg.norm([-0.0106, -1.0, 0.0105])
    got, mv = plane_shift(b64, plane, calib)
    cam = project_velo_to_rect(b64[:, :3], calib)
    cam[:, 1] = (-plane[3] - plane[0] * cam[:, 0] - plane[2] * cam[:, 2]) / plane[1]
    cur = project_rect_to_velo(cam, calib)[:, 2]
    assert np.array_equal(mv, b64[:, 2] - cur)
    assert np.array_equal(got[:, 2], (b64[:, 2] - mv).astype(np.float32))
    assert np.array_equal(got[:, [0, 1, 3, 4, 5, 6]], b64[:, [0, 1, 3, 4, 5, 6]].astype(np.float32))
    assert ((b64[:, 2] - mv) != cur).any(), "some rows tell the subtraction from the assignment"


def test_plane_arguments_are_validated(tree):
    from sassd_b200.augment import PointAugmentor
    from sassd_b200.kitti_data import read_plane
    aug = _augmentor(tree, "car", 0)
    plane, calib = _plane_and_calib(tree, 0)
    none = np.zeros((0, 7), np.float32)
    bad = [dict(road_planes=[plane]), dict(calibs=[calib]),
           dict(road_planes=[plane, plane], calibs=[calib]), dict(road_planes=[plane], calibs=[calib, calib]),
           dict(road_planes=[plane[:3]], calibs=[calib]), dict(road_planes=[np.append(plane, 1.0)], calibs=[calib]),
           dict(road_planes=[[0.0, -1.0, np.nan, 1.6]], calibs=[calib]),
           dict(road_planes=[[0.0, -np.inf, 0.0, 1.6]], calibs=[calib]),
           dict(road_planes=[["0", "-1", "0", "1.6"]], calibs=[calib])]
    for kw in bad:
        with pytest.raises(ValueError, match="road_planes|road plane"):
            aug.augment(None, None, 1, [none], [[]], ["Car"], **kw)
    # valid planes reach the next check: this augmentor has no device database
    with pytest.raises(ValueError, match="without a device database"):
        aug.augment(None, None, 1, [none], [[]], ["Car"], road_planes=[plane], calibs=[calib])
    missing = os.path.join(tree, "training", "planes", "000099.txt")
    with pytest.raises(FileNotFoundError, match="000099.txt"):
        read_plane(missing)
    info = os.path.join(tree, "kitti_dbinfos_train.pkl")
    with pytest.raises(NotImplementedError, match=r"augment\(road_planes=, calibs=\)"):
        PointAugmentor(tree, info, ["Car"], 5, 15, [-1], global_rot_range=[0, 1], center_noise_std=[1, 1, 1],
                       scale_range=[1, 1], device=None, with_plane=True)


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def reduced(tree, tmp_path_factory):
    """The tree after the repo's create_data (velodyne_reduced and gt_database)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from sassd_b200 import create_data as CD
    root = str(tmp_path_factory.mktemp("kitti_plane_cd") / "kitti")
    shutil.copytree(tree, root)
    os.remove(os.path.join(root, "kitti_dbinfos_train.pkl"))
    assert CD.main(["--data-root", root, "--batch", "4"]) == 0
    return root + os.sep


def _run(root, cfg, seed, batch, lidar="velodyne_reduced"):
    import torch
    from sassd_b200 import ops
    from sassd_b200.kitti_data import KittiSplit
    aug = _augmentor(root, cfg, seed, device="cuda")
    split = KittiSplit(root, "train", lidar=lidar)
    ids, res = KR.TRAIN, []
    for i in range(0, len(ids), batch):
        bids = ids[i:i + batch]
        frames = [split.frame(idx) for idx in bids]
        pts = [f[0] for f in frames]
        off = np.concatenate([[0], np.cumsum([len(p) for p in pts])]).astype(np.int32)
        d_pts, d_off = torch.from_numpy(np.concatenate(pts, 0)).cuda(), torch.from_numpy(off).cuda()
        if lidar == "velodyne":
            planes = np.stack([split.planes(f[1]["calib"], f[1]["img_shape"]) for f in frames])
            d_pts, d_off = ops.frustum_crop(d_pts, d_off, len(bids), torch.from_numpy(planes).cuda())
        gts = [_frame(root, idx) for idx in bids]
        road = [_plane_and_calib(root, idx)[0] for idx in bids]
        out, o, boxes, labels, keep, sel = aug.augment(
            d_pts, d_off, len(bids), [g[0] for g in gts], [g[1] for g in gts], CONFIGS[cfg]["class_names"],
            road_planes=road, calibs=[f[1]["calib"] for f in frames])
        host, o = out.cpu().numpy(), o.cpu().numpy()
        for b in range(len(bids)):
            res.append(dict(cloud=host[o[b]:o[b + 1]].copy(), boxes=boxes[b], labels=labels[b], keep=keep[b],
                            sel=sel[b]))
    return res


def _check_run(gold, key, res):
    sels = _split(gold, key, "sel", gold[key + "_nsel"])
    boxes = _split(gold, key, "boxes", gold[key + "_nbox"])
    labels = _split(gold, key, "labels", gold[key + "_nbox"])
    for f, r in enumerate(res):
        assert np.array_equal(r["sel"], sels[f]), (key, f)
        assert np.array_equal(_bits(r["boxes"]), _bits(boxes[f])), (key, f)
        assert np.array_equal(r["labels"], labels[f])
        assert bool(r["keep"]) == bool(gold[key + "_keep"][f])
        full = "%s_cloud%d" % (key, f)
        if full in gold:
            ref = gold[full]
            assert r["cloud"].shape == ref.shape, (f, r["cloud"].shape, ref.shape)
            bad = np.nonzero((r["cloud"].view(np.int32) != ref.view(np.int32)).any(1))[0]
            assert len(bad) == 0, (f, bad[:5], r["cloud"][bad[:3]], ref[bad[:3]])
        assert sha(r["cloud"]) == gold[key + "_cloud_sha"][f], (key, f)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,seed", RUNS)
def test_augment_with_planes_matches_the_reference(gold, reduced, cfg, seed):
    key = "%s_s%d" % (cfg, seed)
    for batch in (1, 4):
        _check_run(gold, key, _run(reduced, cfg, seed, batch))


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,seed", [("car", 0), ("multi", 1)])
def test_full_sweeps_cropped_then_augmented_with_planes_match_the_reference(gold, reduced, cfg, seed):
    _check_run(gold, "%s_s%d" % (cfg, seed), _run(reduced, cfg, seed, 3, lidar="velodyne"))


@pytest.mark.gpu
def test_assemble_rounds_after_the_centre_add_and_again_after_the_move():
    """Hand-made database rows, two records in two frames, no box and an identity frame transform: a row's z is
    (float)((double)(float)((double)z + c) - dz), where a fused single rounding (float)((double)z + c - dz) differs on
    many rows; x and y take only the centre.  Without dz the rows are as before."""
    import torch
    from sassd_b200 import ops
    rng = np.random.default_rng(11)
    n = 4096
    db = np.concatenate([rng.uniform(-2, 2, (n, 3)), rng.random((n, 1))], 1).astype(np.float32)
    ctr = np.array([[15.0, 2.0, -1.0134567891234567], [30.5, -4.25, -0.7890123456789012]])
    dz = np.array([-0.93456789012345678, 0.12345678901234567])
    half = n // 2
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    i32 = lambda v: t(np.array(v, np.int32))  # noqa: E731
    status = torch.zeros((1,), dtype=torch.int32, device="cuda")
    empty = torch.zeros((1, 4), dtype=torch.float32, device="cuda")

    def run(d):
        out, o = ops.augment_assemble(
            empty, i32([0, 0, 0]), 2, i32([0, half, n]), i32([0, half, n]), i32([0, half]), t(ctr), t(db),
            i32([0, 0, 0]), torch.zeros((1, 6, 4), dtype=torch.float32, device="cuda"),
            torch.zeros((1, 3), dtype=torch.float32, device="cuda"), i32([0]),
            torch.zeros((1, 1, 2), dtype=torch.float32, device="cuda"),
            torch.zeros((1, 1, 3), dtype=torch.float64, device="cuda"),
            t(np.array([[0, 1, 0, 0, 1, 1]] * 2, np.float32)), n, status, dz=None if d is None else t(d))
        assert int(status.cpu()) == 0 and list(o.cpu().numpy()) == [0, half, n]
        return out.cpu().numpy()
    rec = np.repeat([0, 1], [half, n - half])
    centred = (db[:, :3].astype(np.float64) + ctr[rec]).astype(np.float32)
    twice = (centred[:, 2].astype(np.float64) - dz[rec]).astype(np.float32)
    fused = (db[:, 2].astype(np.float64) + ctr[rec, 2] - dz[rec]).astype(np.float32)
    assert (twice != fused).sum() > 100, "the rows must tell the two roundings apart"
    got = run(dz)
    assert np.array_equal(got[:, 2].view(np.int32), twice.view(np.int32))
    assert np.array_equal(got[:, :2].view(np.int32), centred[:, :2].view(np.int32))
    assert np.array_equal(got[:, 3].view(np.int32), db[:, 3].view(np.int32))
    assert np.array_equal(run(None)[:, :3].view(np.int32), centred.view(np.int32))


def _plane_cfg(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "configs", "car_cfg.py")) as fh:
        text = fh.read()
    path = str(tmp_path / "car_plane_cfg.py")
    with open(path, "w") as fh:
        fh.write(text + "\ndata['train']['with_plane'] = True\n")
    return path


@pytest.mark.gpu
@pytest.mark.parametrize("lidar", ["velodyne_reduced", "velodyne"])
def test_cli_with_plane_writes_the_reference_clouds(gold, reduced, tmp_path, lidar):
    from sassd_b200 import augment as A
    out = str(tmp_path / "aug")
    assert A.main([_plane_cfg(tmp_path), "--data-root", reduced, "--lidar", lidar, "--seed", "0", "--batch", "4",
                   "--out", out]) == 0
    for f, idx in enumerate(KR.TRAIN):
        with open(os.path.join(out, "%06d.bin" % idx), "rb") as fh:
            assert hashlib.sha256(fh.read()).hexdigest() == gold["car_s0_cloud_sha"][f], idx
        z = np.load(os.path.join(out, "%06d.npz" % idx))
        assert bool(z["keep"]) == bool(gold["car_s0_keep"][f])


@pytest.mark.gpu
def test_cli_with_plane_fails_on_a_missing_plane_file_before_its_batch(reduced, tmp_path):
    from sassd_b200 import augment as A
    root = str(tmp_path / "kitti")
    shutil.copytree(reduced, root)
    missing = os.path.join(root, "training", "planes", "%06d.txt" % KR.TRAIN[4])
    os.remove(missing)
    out = str(tmp_path / "aug")
    with pytest.raises(FileNotFoundError, match=re.escape(missing)):
        A.main([_plane_cfg(tmp_path), "--data-root", root + os.sep, "--lidar", "velodyne_reduced", "--seed", "0",
                "--batch", "4", "--out", out])
    written = sorted(os.listdir(out))
    assert written == sorted("%06d.%s" % (i, e) for i in KR.TRAIN[:4] for e in ("bin", "npz")), written

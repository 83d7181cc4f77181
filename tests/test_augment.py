"""Training-time augmentation (sassd_b200.augment, csrc/augment.cu) against tests/golden/augment.npz, produced by the
reference's own PointAugmentor and prepare_train_img with numba compiled (tests/golden/make_golden_augment.py) on the
synthetic root of tests/kitti_root.py.

Bar: every draw, sampled record, noise index, final box and label, keep flag and augmented-cloud digest identical to
the reference's, at batch 1 and batch 4."""
import hashlib
import os
import pickle
import shutil

import numpy as np
import pytest

from tests import kitti_root as KR
from sassd_b200.augment import rotation_z32

CONFIGS = {
    "car": dict(sample_classes=["Car"], min_num_points=[5], sample_max_num=[15], class_names=["Car"]),
    "multi": dict(sample_classes=["Car", "Pedestrian", "Cyclist"], min_num_points=[5, 0, 0],
                  sample_max_num=[15, 10, 10], class_names=["Car", "Pedestrian", "Cyclist"]),
}
COMMON = dict(removed_difficulties=[-1], global_rot_range=[-0.78539816, 0.78539816],
              gt_rot_range=[-0.78539816, 0.78539816], center_noise_std=[1., 1., .5], scale_range=[0.95, 1.05])
RUNS = [(c, s) for c in CONFIGS for s in (0, 1, 2)]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "augment.npz"))


def _restore(obj):
    """kitti_root.unflatten's (type name, array) leaves back to the pickled objects."""
    if isinstance(obj, dict):
        return {k: _restore(v) for k, v in obj.items()}
    if isinstance(obj, list):
        return [_restore(v) for v in obj]
    kind, a = obj
    if kind == "ndarray":
        return a
    if kind in ("str", "int", "float", "bool"):
        return {"str": str, "int": int, "float": float, "bool": bool}[kind](a[()])
    return a[()]


@pytest.fixture(scope="module")
def tree(tmp_path_factory, golden_dir):
    """The synthetic root with the reference's kitti_dbinfos_train.pkl (from tests/golden/create_data.npz)."""
    cd = np.load(os.path.join(golden_dir, "create_data.npz"))
    root = str(tmp_path_factory.mktemp("kitti_aug") / "kitti")
    KR.write_tree(root)
    with open(os.path.join(root, "kitti_dbinfos_train.pkl"), "wb") as fh:
        pickle.dump(_restore(KR.unflatten(cd, "dbinfos_train")), fh)
    return root


def _augmentor(root, cfg, seed, device=None):
    from sassd_b200.augment import PointAugmentor
    c = dict(CONFIGS[cfg])
    c.pop("class_names")
    return PointAugmentor(root, os.path.join(root, "kitti_dbinfos_train.pkl"), rng=np.random.RandomState(seed),
                          device=device, **c, **COMMON)


def _frame(root, idx):
    from sassd_b200.kitti_data import labelled_boxes, read_label
    from sassd_b200.results import Calibration
    d = os.path.join(root, "training")
    calib = Calibration(os.path.join(d, "calib", "%06d.txt" % idx))
    return labelled_boxes(read_label(os.path.join(d, "label_2", "%06d.txt" % idx)), calib)


def _split(gold, key, name, counts):
    a = gold["%s_%s" % (key, name)]
    off = np.concatenate([[0], np.cumsum(counts)])
    return [a[off[i]:off[i + 1]] for i in range(len(counts))]


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("cfg,seed", RUNS)
def test_host_draws_and_boxes_match_the_reference(gold, tree, cfg, seed):
    aug = _augmentor(tree, cfg, seed)
    key = "%s_s%d" % (cfg, seed)
    sels = _split(gold, key, "sel", gold[key + "_nsel"])
    boxes = _split(gold, key, "boxes", gold[key + "_nbox"])
    labels = _split(gold, key, "labels", gold[key + "_nbox"])
    for f, idx in enumerate(KR.TRAIN):
        gt, names = _frame(tree, idx)
        plan = aug.draw(gt, names, CONFIGS[cfg]["class_names"])
        paths = ";".join(aug.records[r]["path"] for r in plan["records"])
        assert paths == gold[key + "_paths"][f], (key, f)
        assert sha(plan["loc"]) == gold[key + "_loc_sha"][f]
        assert sha(plan["rot"]) == gold[key + "_rot_sha"][f]
        assert (plan["flip"], plan["angle"], plan["scale"]) == (
            bool(gold[key + "_flip"][f]), gold[key + "_angle"][f], gold[key + "_scale"][f])
        assert len(plan["boxes"]) == len(sels[f])
        b, lab = aug.finish_boxes(plan, sels[f])
        assert np.array_equal(b.view(np.int32), boxes[f].view(np.int32)), (key, f)
        assert np.array_equal(lab, labels[f])
        assert (len(b) > 0) == bool(gold[key + "_keep"][f])


def test_collision_restatement_matches_the_compiled_reference(gold):
    from sassd_b200.augment import box_collision
    a, b = gold["coll_a"], gold["coll_b"]
    got = np.array([box_collision(a[i:i + 1], b[i:i + 1])[0, 0] for i in range(len(a))])
    assert np.array_equal(got, gold["coll"])
    got64 = np.array([box_collision(a[i:i + 1].astype(np.float64), b[i:i + 1].astype(np.float64))[0, 0]
                      for i in range(len(a))])
    assert np.array_equal(got64, gold["coll_f64"])
    assert gold["coll"][0] and gold["coll"][1], "a box inside another collides when compiled"


def test_float32_planes_give_the_reference_boundary_masks(gold):
    from sassd_b200.augment import box_planes32
    pl = box_planes32(gold["bnd_boxes"])
    assert pl.dtype == np.float32
    pts = gold["bnd_points"]
    mask = np.unpackbits(gold["bnd_mask"])[:len(pts) * len(pl)].reshape(len(pl), len(pts)).astype(bool)
    with np.errstate(invalid="ignore", over="ignore"):
        for j in range(len(pl)):
            s = np.zeros(len(pts), bool)
            for k in range(6):
                v = pts[:, 0] * pl[j, k, 0] + pts[:, 1] * pl[j, k, 1] + pts[:, 2] * pl[j, k, 2] + pl[j, k, 3]
                s |= v >= 0
            assert np.array_equal(~s, mask[j])


def test_argument_and_config_validation(tree):
    from sassd_b200 import Config
    from sassd_b200.augment import PointAugmentor
    info = os.path.join(tree, "kitti_dbinfos_train.pkl")
    with pytest.raises(ValueError, match="no Tram records"):
        PointAugmentor(tree, info, ["Tram"], 5, 15, [-1], global_rot_range=[0, 1], center_noise_std=[1, 1, 1],
                       scale_range=[1, 1], device=None)
    with pytest.raises(NotImplementedError):
        PointAugmentor(tree, info, ["Car"], 5, 15, [-1], global_rot_range=[0, 1], center_noise_std=[1, 1, 1],
                       scale_range=[1, 1], device=None, with_plane=True)
    with pytest.raises(ValueError, match="one entry per sample class"):
        PointAugmentor(tree, info, ["Car"], [5, 5], 15, [-1], global_rot_range=[0, 1], center_noise_std=[1, 1, 1],
                       scale_range=[1, 1], device=None)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for name, classes, nums in (("car_cfg", ["Car"], [15]), ("multi_cfg", ["Car", "Pedestrian", "Cyclist"],
                                                              [15, 10, 10])):
        cfg = Config.fromfile(os.path.join(root, "configs", name + ".py"))
        a = cfg.data["train"]["augmentor"]
        assert a["sample_classes"] == classes and a["sample_max_num"] == nums
        assert cfg.data["train"]["class_names"] == cfg.data["val"]["class_names"]


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def reduced(tree, tmp_path_factory):
    """The tree after the repo's create_data (velodyne_reduced and gt_database)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from sassd_b200 import create_data as CD
    root = str(tmp_path_factory.mktemp("kitti_aug_cd") / "kitti")
    shutil.copytree(tree, root)
    os.remove(os.path.join(root, "kitti_dbinfos_train.pkl"))
    assert CD.main(["--data-root", root, "--batch", "4"]) == 0
    return root + os.sep


def _run(root, cfg, seed, batch, ids, lidar="velodyne_reduced"):
    import torch
    from sassd_b200 import ops
    from sassd_b200.kitti_data import KittiSplit
    aug = _augmentor(root, cfg, seed, device="cuda")
    split = KittiSplit(root, "train", lidar=lidar)
    res = []
    for i in range(0, len(ids), batch):
        bids = ids[i:i + batch]
        frames = [split.frame(idx) for idx in bids]
        pts = [f[0] for f in frames]
        off = np.concatenate([[0], np.cumsum([len(p) for p in pts])]).astype(np.int32)
        d_pts = torch.from_numpy(np.concatenate(pts, 0)).cuda()
        d_off = torch.from_numpy(off).cuda()
        if lidar == "velodyne":
            planes = np.stack([split.planes(f[1]["calib"], f[1]["img_shape"]) for f in frames])
            d_pts, d_off = ops.frustum_crop(d_pts, d_off, len(bids), torch.from_numpy(planes).cuda())
        gts = [_frame(root, idx) for idx in bids]
        out, o, boxes, labels, keep, sel = aug.augment(d_pts, d_off, len(bids), [g[0] for g in gts],
                                                       [g[1] for g in gts], CONFIGS[cfg]["class_names"])
        host, o = out.cpu().numpy(), o.cpu().numpy()
        for b in range(len(bids)):
            res.append(dict(cloud=host[o[b]:o[b + 1]].copy(), boxes=boxes[b], labels=labels[b], keep=keep[b],
                            sel=sel[b]))
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,seed", RUNS)
def test_augment_matches_the_reference(gold, reduced, cfg, seed):
    key = "%s_s%d" % (cfg, seed)
    sels = _split(gold, key, "sel", gold[key + "_nsel"])
    boxes = _split(gold, key, "boxes", gold[key + "_nbox"])
    labels = _split(gold, key, "labels", gold[key + "_nbox"])
    runs = {B: _run(reduced, cfg, seed, B, KR.TRAIN) for B in (1, 4)}
    for f in range(len(KR.TRAIN)):
        r = runs[1][f]
        assert np.array_equal(r["sel"], sels[f]), (key, f)
        assert np.array_equal(r["boxes"].view(np.int32), boxes[f].view(np.int32)), (key, f)
        assert np.array_equal(r["labels"], labels[f])
        assert bool(r["keep"]) == bool(gold[key + "_keep"][f])
        if f < 2 and seed == 0 and cfg == "car":
            ref = gold["%s_cloud%d" % (key, f)]
            assert r["cloud"].shape == ref.shape
            bad = np.nonzero((r["cloud"].view(np.int32) != ref.view(np.int32)).any(1))[0]
            assert len(bad) == 0, (f, bad[:5], r["cloud"][bad[:3]], ref[bad[:3]])
        assert sha(r["cloud"]) == gold[key + "_cloud_sha"][f], (key, f)
        r4 = runs[4][f]
        assert np.array_equal(r4["cloud"].view(np.int32), r["cloud"].view(np.int32))
        assert np.array_equal(r4["boxes"].view(np.int32), r["boxes"].view(np.int32))


@pytest.mark.gpu
def test_full_sweeps_cropped_then_augmented_match_the_reduced_clouds(reduced):
    a = _run(reduced, "multi", 1, 3, KR.TRAIN, lidar="velodyne")
    b = _run(reduced, "multi", 1, 3, KR.TRAIN)
    for x, y in zip(a, b):
        assert np.array_equal(x["cloud"].view(np.int32), y["cloud"].view(np.int32))
        assert np.array_equal(x["boxes"].view(np.int32), y["boxes"].view(np.int32))


@pytest.mark.gpu
def test_noise_search_kernel_on_adversarial_boxes(gold):
    import torch
    from sassd_b200 import augment as A
    from sassd_b200 import ops
    boxes = gold["ns_boxes"]
    trig = np.array([[A._libm.cosf(float(a)), A._libm.sinf(float(a))] for a in boxes[:, 4]], np.float32)
    rot = gold["ns_rot"]
    try_trig = np.stack([np.cos(rot), np.sin(rot)], -1).astype(np.float32)
    status = torch.zeros((1,), dtype=torch.int32, device="cuda")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    # one frame of all four boxes, then boxes 0-1 and 2-3 as two frames: the fixture's boxes 2 and 3 never meet boxes 0
    # and 1, so each frame's search gives the same tries
    for split in ([0, 4], [0, 2, 4]):
        sel = ops.augment_noise_search(t(boxes), t(trig), t(np.array(split, np.int32)), len(split) - 1, t(try_trig),
                                       t(gold["ns_loc"]), status)
        assert np.array_equal(sel.cpu().numpy(), gold["ns_sel"]), split
    assert (gold["ns_sel"][:2] == -1).all()
    assert int(status.cpu()) == 0


def _search(boxes5, loc, rot, box_off):
    import torch
    from sassd_b200 import augment as A
    from sassd_b200 import ops
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    trig = np.array([[A._libm.cosf(float(a)), A._libm.sinf(float(a))] for a in boxes5[:, 4]], np.float32)
    status = torch.zeros((1,), dtype=torch.int32, device="cuda")
    sel = ops.augment_noise_search(t(boxes5), t(trig), t(np.array(box_off, np.int32)), len(box_off) - 1,
                                   t(np.stack([np.cos(rot), np.sin(rot)], -1).astype(np.float32)), t(loc), status)
    return sel.cpu().numpy(), int(status.cpu())


@pytest.mark.gpu
def test_noise_search_at_the_gt_cap():
    """256 boxes in one frame, the shared-memory capacity: 254 unit boxes 10 m apart find their first try, and the last
    two, a unit box inside a diamond, collide on every small try.  One box more sets GT_CAP and gets no try."""
    from sassd_b200.lib import FLAGS, GT_CAP_MAX
    rng = np.random.RandomState(7)
    g = np.arange(GT_CAP_MAX - 2)
    boxes = np.stack([10.0 * (g % 16), 10.0 * (g // 16), np.ones_like(g), np.ones_like(g), np.zeros_like(g)], 1)
    boxes = np.concatenate([boxes, [[200, 200, 1, 1, 0], [200, 200, 2, 2, np.pi / 4]]]).astype(np.float32)
    loc = rng.normal(scale=0.05, size=[len(boxes), 100, 3])
    rot = rng.uniform(-0.05, 0.05, size=[len(boxes), 100])
    sel, status = _search(boxes, loc, rot, [0, len(boxes)])
    assert status == 0
    assert (sel[:-2] == 0).all() and (sel[-2:] == -1).all()
    extra = np.concatenate([boxes, [[500, 500, 1, 1, 0]]]).astype(np.float32)
    sel, status = _search(extra, np.concatenate([loc, loc[:1]]), np.concatenate([rot, rot[:1]]), [0, len(extra)])
    assert FLAGS[status] == "GT_CAP"
    assert (sel[:-3] == 0).all() and (sel[-3:] == -1).all()


@pytest.mark.gpu
def test_assemble_moves_each_point_by_its_first_box(gold):
    """The point pass on the boundary cloud: every box has one try (no rotation, x moved by 1000 (k + 1)) and the frame
    no flip, rotation or scaling, so a point's x tells which box took it: the first box whose float32 planes contain
    it, as the reference's masks say, after the -centre, +centre round trip."""
    import torch
    from sassd_b200 import ops
    from sassd_b200.augment import box_planes32
    pts, bb = gold["bnd_points"], gold["bnd_boxes"]
    mask = np.unpackbits(gold["bnd_mask"])[:len(pts) * len(bb)].reshape(len(bb), len(pts)).astype(bool)
    n, k = len(pts), len(bb)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    i32 = lambda v: t(np.array(v, np.int32))  # noqa: E731
    loc = np.zeros((k, 1, 3))
    loc[:, 0, 0] = 1000.0 * (np.arange(k) + 1)
    status = torch.zeros((1,), dtype=torch.int32, device="cuda")
    out, o = ops.augment_assemble(
        t(pts), i32([0, n]), 1, i32([0, 0]), i32([0]), i32([]), t(np.zeros((1, 3))), t(np.zeros((1, 4), np.float32)),
        i32([0, k]), t(box_planes32(bb)), t(bb[:, :3]), i32([0] * k), t(np.tile([[[1.0, 0.0]]], (k, 1, 1)).astype(
            np.float32)), t(loc), t(np.array([[0, 1, 0, 0, 1, 1]], np.float32)), n, status)
    assert int(status.cpu()) == 0 and list(o.cpu().numpy()) == [0, n]
    got = out.cpu().numpy()
    first = np.where(mask.any(0), mask.argmax(0), -1)
    exp = pts.copy()
    with np.errstate(invalid="ignore", over="ignore"):
        for j in range(k):
            r = first == j
            c = bb[j, :3]
            exp[r, :3] = (pts[r, :3] - c) + c
            exp[r, 0] = (exp[r, 0].astype(np.float64) + loc[j, 0, 0]).astype(np.float32)
    finite = np.isfinite(pts[:, :3]).all(1)
    assert np.array_equal(got[finite].view(np.int32), exp[finite].view(np.int32))
    assert (~np.isfinite(got[~finite, :3]).all(1)).all()
    assert np.array_equal(got[:, 3].view(np.int32), pts[:, 3].view(np.int32))


@pytest.mark.gpu
def test_drop_kernel_on_boundary_points(gold):
    import torch
    from sassd_b200 import ops
    from sassd_b200.augment import box_planes32
    pts, bb = gold["bnd_points"], gold["bnd_boxes"]
    mask = np.unpackbits(gold["bnd_mask"])[:len(pts) * len(bb)].reshape(len(bb), len(pts)).astype(bool)
    pl = torch.from_numpy(box_planes32(bb)).cuda()
    n = len(pts)
    # frame 0: every box; frame 1: no box; frame 2: empty
    d_pts = torch.from_numpy(np.concatenate([pts, pts], 0)).cuda()
    off = torch.tensor([0, n, 2 * n, 2 * n], dtype=torch.int32, device="cuda")
    box_off = torch.tensor([0, len(bb), len(bb), len(bb)], dtype=torch.int32, device="cuda")
    out, o = ops.augment_drop_points(d_pts, off, 3, pl, box_off)
    o = o.cpu().numpy()
    keep = ~mask.any(0)
    assert list(o) == [0, keep.sum(), keep.sum() + n, keep.sum() + n]
    got = out.cpu().numpy()
    assert np.array_equal(got[:o[1]].view(np.int32), pts[keep].view(np.int32))
    assert np.array_equal(got[o[1]:o[2]].view(np.int32), pts.view(np.int32))


@pytest.mark.gpu
def test_empty_frames_and_capacity_overflow(reduced):
    import torch
    from sassd_b200.lib import SassdError
    aug = _augmentor(reduced, "car", 0, device="cuda")
    # an empty frame with no GT (it still receives samples) and a frame with points and no GT
    pts = torch.from_numpy(np.random.default_rng(0).uniform(0, 10, (64, 4)).astype(np.float32)).cuda()
    off = torch.tensor([0, 0, 64], dtype=torch.int32, device="cuda")
    none = np.zeros((0, 7), np.float32)
    out, o, boxes, labels, keep, sel = aug.augment(pts, off, 2, [none, none], [[], []], ["Car"])
    o = o.cpu().numpy()
    assert o[0] == 0 and o[2] >= o[1] >= 0
    assert torch.isfinite(out[:o[2]]).all()
    for b in range(2):
        assert len(boxes[b]) == len(labels[b]) and keep[b] == (len(boxes[b]) > 0)
    with pytest.raises(SassdError, match="POINTS_CAP"):
        aug.augment(pts, off, 2, [none, none], [[], []], ["Car"], max_points=8)
    too_many = np.tile(np.array([[10, 0, -1, 1.6, 3.9, 1.5, 0]], np.float32), (300, 1))
    with pytest.raises(ValueError, match="at most 256"):
        aug.augment(pts, off, 2, [too_many, none], [["Car"] * 300, []], ["Car"])


def _nothing_sampled(root, device):
    from sassd_b200.augment import PointAugmentor
    return PointAugmentor(root, os.path.join(root, "kitti_dbinfos_train.pkl"), ["Car"], [5], [0], [-1],
                          rng=np.random.RandomState(4), device=device, **{k: v for k, v in COMMON.items()
                                                                          if k != "removed_difficulties"})


@pytest.mark.gpu
def test_frame_without_gt_or_samples_takes_only_the_global_transforms(reduced):
    """sample_max_num 0 and no GT: nothing is pasted or dropped, no box moves a point, and the cloud is the input
    flipped, rotated and scaled as numpy does it on the host."""
    import torch
    aug = _nothing_sampled(reduced, "cuda")
    host = _nothing_sampled(reduced, None)
    pts = np.random.default_rng(1).uniform(-30, 60, (3000, 4)).astype(np.float32)
    none = np.zeros((0, 7), np.float32)
    for _ in range(4):      # frames with and without the flip
        plan = host.draw(none, [], ["Car"])
        out, o, boxes, labels, keep, sel = aug.augment(torch.from_numpy(pts).cuda(), torch.tensor(
            [0, len(pts)], dtype=torch.int32, device="cuda"), 1, [none], [[]], ["Car"])
        assert list(o.cpu().numpy()) == [0, len(pts)]
        assert len(boxes[0]) == 0 and not keep[0] and len(sel[0]) == 0
        exp = pts.copy()
        if plan["flip"]:
            exp[:, 1] = -exp[:, 1]
        exp[:, :3] = exp[:, :3] @ rotation_z32(plan["angle"])
        exp[:, :3] *= plan["scale"]
        assert np.array_equal(out[:len(pts)].cpu().numpy().view(np.int32), exp.view(np.int32))


@pytest.mark.gpu
def test_a_frame_at_the_gt_cap_augments_cleanly(reduced):
    """256 Car boxes (more than sample_max_num, so nothing is sampled) fill the noise search's capacity."""
    import torch
    aug = _augmentor(reduced, "car", 3, device="cuda")
    g = np.arange(256)
    gt = np.stack([5.0 + 4.0 * (g % 16), -35.0 + 4.5 * (g // 16), np.full(256, -1.7), np.full(256, 1.6),
                   np.full(256, 3.9), np.full(256, 1.56), np.zeros(256)], 1).astype(np.float32)
    pts = np.random.default_rng(2).uniform([0, -40, -3, 0], [70, 40, 1, 1], (20000, 4)).astype(np.float32)
    out, o, boxes, labels, keep, sel = aug.augment(torch.from_numpy(pts).cuda(), torch.tensor(
        [0, len(pts)], dtype=torch.int32, device="cuda"), 1, [gt], [["Car"] * 256], ["Car"])
    assert len(sel[0]) == 256 and ((sel[0] >= -1) & (sel[0] < 100)).all()
    assert list(o.cpu().numpy()) == [0, len(pts)]
    assert torch.isfinite(out[:len(pts)]).all()
    assert keep[0] and len(boxes[0]) == len(labels[0]) <= 256


def _synthetic_checkpoint(path):
    from sassd_b200 import checkpoint
    from tests.test_point_aux import _aux_weights
    sd = checkpoint.make_synthetic_state_dict(0, 1)
    sd.update(_aux_weights())
    checkpoint.save_checkpoint(sd, path)
    return path


@pytest.mark.gpu
def test_augmented_batches_through_loss_points(reduced, tmp_path, capsys):
    """An augmented batch's kept frames go through loss_points with finite losses and a clean status (it raises on a
    status bit); the driver's --checkpoint prints the means of the same losses."""
    import torch
    import sassd_b200 as S
    from sassd_b200 import augment as A
    from sassd_b200 import ops
    from sassd_b200.checkpoint import load_params_from_file
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg_path = os.path.join(root, "configs", "car_cfg.py")
    ckpt = _synthetic_checkpoint(str(tmp_path / "synthetic.pth"))
    model, _, _ = S.build_from_config(S.Config.fromfile(cfg_path))
    load_params_from_file(model, ckpt)
    model.eval()
    res = _run(reduced, "car", 0, 4, KR.TRAIN)
    frames = [r for r in res if r["keep"]]
    assert frames
    losses = model.loss_points([r["cloud"] for r in frames], [r["boxes"] for r in frames],
                               [r["labels"] for r in frames])
    assert set(losses) == set(ops.LOSS_KEYS)
    assert all(np.isfinite(v) for v in losses.values()), losses
    assert losses["rpn_loc_loss"] > 0
    capsys.readouterr()
    assert A.main([cfg_path, "--data-root", reduced, "--lidar", "velodyne_reduced", "--seed", "0", "--batch", "4",
                   "--checkpoint", ckpt]) == 0
    line = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("losses over")]
    assert len(line) == 1 and "losses over 2 augmented batches" in line[0]
    vals = dict(kv.rsplit(" ", 1) for kv in line[0].split(": ", 1)[1].split(", "))
    assert set(vals) == set(ops.LOSS_KEYS) and all(np.isfinite(float(v)) for v in vals.values())
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_cli_writes_the_reference_clouds(gold, reduced, tmp_path):
    from sassd_b200 import augment as A
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "aug")
    assert A.main([os.path.join(root, "configs", "car_cfg.py"), "--data-root", reduced, "--lidar",
                   "velodyne_reduced", "--seed", "0", "--batch", "4", "--out", out]) == 0
    for f, idx in enumerate(KR.TRAIN):
        with open(os.path.join(out, "%06d.bin" % idx), "rb") as fh:
            assert hashlib.sha256(fh.read()).hexdigest() == gold["car_s0_cloud_sha"][f]

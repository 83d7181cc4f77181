"""Preparing a KITTI root (python -m sassd_b200.create_data; csrc/frustum.cu sassd_points_in_rbboxes) against
tests/golden/create_data.npz, produced by the reference's own tools/create_data.py on the synthetic root of
tests/kitti_root.py (tests/golden/make_golden_create_data.py).

Bar: box planes bit-identical to the reference's; memberships, counts, offsets and gathered rows bit-identical to the
numpy restatement (oracle.frustum.inside_frustum on each box's planes); every reduced cloud and database file
byte-identical to the reference's, and the info and dbinfo pickles equal field by field, with their types."""
import ctypes
import os
import pickle
import shutil

import numpy as np
import pytest
import torch

from oracle.frustum import inside_frustum
from tests import kitti_root as KR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "create_data.npz"))


@pytest.fixture(scope="module")
def tree(tmp_path_factory, gold):
    """The synthetic root, rebuilt and checked against the digests of the tree the reference ran on."""
    root = str(tmp_path_factory.mktemp("kitti") / "kitti")
    KR.write_tree(root)
    files = sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)
    assert files == list(gold["input_files"])
    assert [KR.file_digest(os.path.join(root, f)) for f in files] == list(gold["input_sha"]), "tree writer drifted"
    return root


def _copy(tree, dst):
    shutil.copytree(tree, dst)
    return str(dst)


def _boundary(z):
    boxes, pts = z["boundary_boxes"], z["boundary_points"]
    mask = np.unpackbits(z["boundary_mask"])[:len(boxes) * len(pts)].reshape(len(boxes), len(pts)).astype(bool)
    return boxes, pts, mask


def _members(points, boxes):
    """numpy restatement: per box, the member rows relative to its centre, (float32)(float64(p) - c)."""
    from sassd_b200.create_data import box_planes
    planes = box_planes(boxes) if len(boxes) else np.zeros((0, 6, 4))
    out = []
    for p, b in zip(planes, boxes):
        rows = points[inside_frustum(points, p)].copy()
        with np.errstate(invalid="ignore"):
            rows[:, :3] -= b[:3]
        out.append(rows)
    return out


# ------------------------------------------------------------------ CPU
def test_box_planes_are_the_reference_planes_bit_for_bit(gold):
    from sassd_b200.create_data import box_planes
    got = box_planes(gold["boxes"])
    assert got.dtype == np.float64 and got.shape == gold["box_planes"].shape
    assert np.array_equal(got.view(np.uint64), gold["box_planes"].view(np.uint64))


def test_numpy_restatement_reproduces_the_reference_boundary_masks(gold):
    from sassd_b200.create_data import box_planes
    boxes, pts, mask = _boundary(gold)
    planes = box_planes(boxes)
    for j in range(len(boxes)):
        assert np.array_equal(inside_frustum(pts, planes[j]), mask[j]), j
    # the cloud straddles the faces, and a zero-height box holds only non-finite rows
    assert 0.1 < mask[0].mean() < 0.9
    assert (~np.isfinite(pts[mask[2], :3])).any(axis=1).all()


def test_infos_equal_the_reference_infos(gold, tree):
    """Info dicts of the product's host code, with num_points_in_gt from the numpy restatement."""
    from sassd_b200 import create_data as CD
    from sassd_b200.frustum import camera_frustum_planes
    from sassd_b200.kitti_data import read_split
    from sassd_b200.results import Calibration
    infos = {}
    for split in CD.SPLITS:
        infos[split] = []
        for idx in read_split(tree, split):
            info, pts = CD.frame_info(tree, idx, split != "test")
            calib = Calibration({"P2": info["calib/P2"][:3], "Tr_velo_to_cam": info["calib/Tr_velo_to_cam"][:3],
                                 "R0_rect": info["calib/R0_rect"][:3, :3]})
            cropped = pts[inside_frustum(pts, camera_frustum_planes(calib, info["img_shape"]))]
            if "annos" in info:
                boxes = CD.lidar_boxes(info["annos"], info["calib/R0_rect"], info["calib/Tr_velo_to_cam"])
                CD.num_points_in_gt(info["annos"], np.array([len(m) for m in _members(cropped, boxes)], np.int64))
            infos[split].append(info)
    infos["trainval"] = infos["train"] + infos["val"]
    for split in ("train", "val", "trainval", "test"):
        KR.assert_same(KR.leaves(infos[split]), KR.unflatten(gold, "infos_" + split), split)
    npts = np.concatenate([i["annos"]["num_points_in_gt"] for i in infos["trainval"]])
    assert (npts == -1).sum() > 0 and (npts == 0).sum() > 0 and (npts > 0).sum() > 10


@pytest.mark.parametrize("argv, message", [
    (["--db-split", "val"], "invalid choice"),
    (["--batch", "0"], "--batch"),
    (["--classes", "Car", "Bus"], "unknown --classes"),
])
def test_cli_rejects_bad_arguments(tree, argv, message, capsys):
    from sassd_b200 import create_data as CD
    with pytest.raises(SystemExit):
        CD.parse_args(["--data-root", tree] + argv)
    assert message in capsys.readouterr().err


def test_cli_rejects_a_missing_image_set(tree, tmp_path, capsys):
    from sassd_b200 import create_data as CD
    root = _copy(tree, tmp_path / "kitti")
    os.remove(os.path.join(root, "ImageSets", "val.txt"))
    with pytest.raises(SystemExit):
        CD.parse_args(["--data-root", root])
    assert "val.txt not found" in capsys.readouterr().err


def test_rbboxes_symbols_and_argument_validation():
    from sassd_b200 import lib as L
    lib = L.load()
    assert "sassd_points_in_rbboxes" in L.exported_symbols()
    assert lib.sassd_points_in_rbboxes_workspace_bytes(1000, 1, 1) == 8
    assert lib.sassd_points_in_rbboxes_workspace_bytes(1 << 20, 16, 64) == 8 * 16 * 64
    a, b = ctypes.c_void_p(8), ctypes.c_void_p(16)     # never dereferenced on these paths
    ws = 1 << 20
    f = lib.sassd_points_in_rbboxes
    ok = [a, a, 100, 2, a, a, a, 4, a, a, b, 10, a, a, ws, None]
    for k in (0, 1, 4, 5, 6, 8, 9, 12, 13):      # every required pointer
        args = list(ok)
        args[k] = None
        assert f(*args) == -1, k
    for k, v in ((3, 0), (3, 257), (2, -1), (7, 0), (7, 257), (11, -1)):
        args = list(ok)
        args[k] = v
        assert f(*args) == -1, (k, v)
    args = list(ok); args[10] = None                 # no gather buffer needs gather_cap 0
    assert f(*args) == -1
    args = list(ok); args[10] = a                    # gathered onto the points
    assert f(*args) == -1
    args = list(ok); args[14] = 8                    # workspace too small
    assert f(*args) == -3


# ------------------------------------------------------------------ GPU: the kernel
def _frames_case(z, tree, B):
    """B frames with their LiDAR boxes: the boundary cloud, full sweeps of the tree with their label boxes (and the
    overlapping pair, the box behind the camera, the zero-height box), a frame without boxes and an empty frame."""
    from sassd_b200 import create_data as CD
    bboxes, bnd, _ = _boundary(z)
    pool = [(bnd, bboxes)]
    for idx in (0, 1, 2, 5):
        info, pts = CD.frame_info(tree, idx, True)
        pool.append((pts, CD.lidar_boxes(info["annos"], info["calib/R0_rect"], info["calib/Tr_velo_to_cam"])))
    pool.append((pool[1][0][::3].copy(), np.zeros((0, 7))))
    pool.append((np.zeros((0, 4), np.float32), pool[2][1]))
    if B == 1:
        return [pool[0]]
    return [pool[(3 * b + 1) % len(pool)] for b in range(B - 2)] + [pool[-1], pool[0]]


def _run(frames, dev, gather_cap=None, box_cap=None, ws=None):
    from sassd_b200 import create_data as CD
    from sassd_b200 import ops
    B = len(frames)
    off = np.concatenate([[0], np.cumsum([len(p) for p, _ in frames])]).astype(np.int32)
    box_cap = box_cap or max(1, max(len(b) for _, b in frames))
    planes = np.zeros((B, box_cap, 6, 4))
    centres = np.zeros((B, box_cap, 3))
    for i, (_, bx) in enumerate(frames):
        n = min(len(bx), box_cap)
        if n:
            planes[i, :n] = CD.box_planes(bx[:n])
            centres[i, :n] = bx[:n, :3]
    nbox = np.array([len(b) for _, b in frames], np.int32)
    pts = np.concatenate([p for p, _ in frames] + [np.zeros((1, 4), np.float32)], 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)    # noqa: E731
    cap = int(off[-1]) * 2 if gather_cap is None else gather_cap
    return ops.points_in_rbboxes(t(pts), t(off), B, t(planes), t(centres), t(nbox), cap, ws=ws)


def _check(frames, counts, seg_off, gathered):
    counts, seg_off, gathered = counts.cpu().numpy(), seg_off.cpu().numpy(), gathered.cpu().numpy()
    box_cap = counts.shape[1]
    exp_counts = np.zeros_like(counts)
    rows = []
    for b, (p, bx) in enumerate(frames):
        m = _members(p, bx)
        exp_counts[b, :len(m)] = [len(r) for r in m]
        rows.append(m)
    np.testing.assert_array_equal(counts, exp_counts)
    np.testing.assert_array_equal(seg_off, np.concatenate([[0], np.cumsum(exp_counts.reshape(-1))]))
    for b, m in enumerate(rows):
        for j, r in enumerate(m):
            q = b * box_cap + j
            got = gathered[seg_off[q]:seg_off[q + 1]]
            assert got.tobytes() == np.ascontiguousarray(r).tobytes(), (b, j)
    return exp_counts


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2, 9])
def test_kernel_matches_the_reference_masks_and_the_restatement(gold, tree, B):
    dev = torch.device("cuda:0")
    frames = _frames_case(gold, tree, B)
    counts, seg_off, gathered, status = _run(frames, dev)
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    exp = _check(frames, counts, seg_off, gathered)
    # the boundary cloud's counts are the reference's own points_in_rbbox masks
    bboxes, _, mask = _boundary(gold)
    np.testing.assert_array_equal(exp[-1, :len(bboxes)], mask.sum(1))      # the last frame is the boundary cloud
    if B > 2:
        assert (exp[:-2].sum(1) > 0).any(), "no member in the sweeps"


@pytest.mark.gpu
def test_capacity_overflows_set_the_status_and_raise(gold, tree):
    from sassd_b200 import lib as L
    dev = torch.device("cuda:0")
    frames = _frames_case(gold, tree, 4)
    counts, seg_off, gathered, status = _run(frames, dev)
    total = int(seg_off[-1])
    c2, s2, g2, st2 = _run(frames, dev, gather_cap=total - 7)
    torch.cuda.synchronize()
    assert int(st2.item()) == L.GATHER_CAP
    assert torch.equal(c2, counts) and torch.equal(s2, seg_off)     # counts and offsets stay exact
    assert torch.equal(g2[:total - 7].view(torch.int32), gathered[:total - 7].view(torch.int32))   # rows that fit
    with pytest.raises(L.SassdError, match="GATHER_CAP"):
        L.raise_on_status(st2)
    # more boxes than box_cap: the first box_cap are used
    n = max(len(b) for _, b in frames)
    c3, _, _, st3 = _run(frames, dev, box_cap=n - 1)
    torch.cuda.synchronize()
    assert int(st3.item()) == 64
    np.testing.assert_array_equal(c3.cpu().numpy(), counts.cpu().numpy()[:, :n - 1])


@pytest.mark.gpu
def test_captured_call_gives_the_eager_bytes(gold, tree):
    from sassd_b200 import create_data as CD
    from sassd_b200 import ops
    dev = torch.device("cuda:0")
    B, box_cap, n_cap, gcap = 3, 20, 3 * 131072, 3 * 131072
    pts = torch.zeros((n_cap, 4), dtype=torch.float32, device=dev)
    off = torch.zeros((B + 1,), dtype=torch.int32, device=dev)
    planes = torch.zeros((B, box_cap, 6, 4), dtype=torch.float64, device=dev)
    centres = torch.zeros((B, box_cap, 3), dtype=torch.float64, device=dev)
    nbox = torch.zeros((B,), dtype=torch.int32, device=dev)
    status = torch.zeros((1,), dtype=torch.int32, device=dev)
    ws = ops.Workspace()
    pool = _frames_case(gold, tree, 9)

    def load(frames):
        n = [len(p) for p, _ in frames]
        pts.zero_()
        pts[:sum(n)].copy_(torch.from_numpy(np.concatenate([p for p, _ in frames], 0)))
        off.copy_(torch.from_numpy(np.concatenate([[0], np.cumsum(n)]).astype(np.int32)))
        pl, ce = np.zeros((B, box_cap, 6, 4)), np.zeros((B, box_cap, 3))
        for i, (_, bx) in enumerate(frames):
            if len(bx):
                pl[i, :len(bx)], ce[i, :len(bx)] = CD.box_planes(bx), bx[:, :3]
        planes.copy_(torch.from_numpy(pl)); centres.copy_(torch.from_numpy(ce))
        nbox.copy_(torch.from_numpy(np.array([len(b) for _, b in frames], np.int32)))

    load(pool[:3])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.points_in_rbboxes(pts, off, B, planes, centres, nbox, gcap, status=status, ws=ws)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        g_out = ops.points_in_rbboxes(pts, off, B, planes, centres, nbox, gcap, status=status, ws=ws)
    for sel in ([4, 0, 6], [1, 2, 7], [0, 0, 3]):
        frames = [pool[i] for i in sel]
        load(frames)
        g.replay()
        e_counts, e_off, e_rows, e_status = ops.points_in_rbboxes(pts, off, B, planes, centres, nbox, gcap)
        torch.cuda.synchronize()
        assert int(status.item()) == 0 and int(e_status.item()) == 0
        assert torch.equal(g_out[0], e_counts) and torch.equal(g_out[1], e_off)
        n = int(e_off[-1])
        assert n > 0 and g_out[2][:n].cpu().numpy().tobytes() == e_rows[:n].cpu().numpy().tobytes()
        _check(frames, e_counts, e_off, e_rows)


# ------------------------------------------------------------------ GPU: the driver
def _outputs(root, db_split="train"):
    files = KR.output_files(root)
    pk = {}
    for name in ["kitti_infos_%s" % s for s in ("train", "val", "trainval", "test")] + ["kitti_dbinfos_" + db_split]:
        with open(os.path.join(root, name + ".pkl"), "rb") as fh:
            pk[name] = pickle.load(fh)
    return files, {f: KR.file_digest(os.path.join(root, f)) for f in files}, pk


@pytest.mark.gpu
def test_driver_writes_the_reference_files(gold, tree, tmp_path):
    from sassd_b200 import create_data as CD
    runs = {}
    for batch in (16, 1, 4):
        root = _copy(tree, tmp_path / ("b%d" % batch))
        assert CD.main(["--data-root", root, "--batch", str(batch), "--workers", "3"]) == 0
        runs[batch] = _outputs(root)
    files, sha, pk = runs[16]
    assert files == list(gold["files_train"])
    assert [sha[f] for f in files] == list(gold["files_sha_train"])
    for s in ("train", "val", "trainval", "test"):
        KR.assert_same(KR.leaves(pk["kitti_infos_" + s]), KR.unflatten(gold, "infos_" + s), s)
    KR.assert_same(KR.leaves(pk["kitti_dbinfos_train"]), KR.unflatten(gold, "dbinfos_train"), "dbinfos")
    assert sum(len(v) for v in pk["kitti_dbinfos_train"].values()) > 20
    for batch in (1, 4):
        assert runs[batch][:2] == runs[16][:2], batch
        for k in pk:
            KR.assert_same(KR.leaves(runs[batch][2][k]), KR.leaves(pk[k]), "%s batch %d" % (k, batch))

    root = _copy(tree, tmp_path / "tv")
    assert CD.main(["--data-root", root, "--db-split", "trainval", "--batch", "3"]) == 0
    files, sha, pk = _outputs(root, "trainval")
    db = [f for f in files if f.startswith("gt_database/")]
    assert db == list(gold["files_trainval"])
    assert [sha[f] for f in db] == list(gold["files_sha_trainval"])
    KR.assert_same(KR.leaves(pk["kitti_dbinfos_trainval"]), KR.unflatten(gold, "dbinfos_trainval"), "dbinfos tv")


@pytest.mark.gpu
def test_detection_reads_the_reduced_clouds_it_wrote(tree, tmp_path):
    """python -m sassd_b200.test --lidar velodyne_reduced on the written clouds gives the result files of the device
    crop of the full sweeps."""
    from sassd_b200 import checkpoint
    from sassd_b200 import create_data as CD
    from sassd_b200 import test as T
    root = _copy(tree, tmp_path / "kitti")
    CD.main(["--data-root", root, "--classes", "Car"])
    ckpt = str(tmp_path / "synthetic.pth")
    checkpoint.save_checkpoint(checkpoint.make_synthetic_state_dict(0, 1), ckpt)
    cfg = os.path.join(ROOT, "configs", "car_cfg.py")
    outs = {}
    for lidar in ("velodyne", "velodyne_reduced"):
        out = str(tmp_path / lidar)
        res = T.run(T.parse_args([cfg, ckpt, "--data-root", root, "--split", "train", "--batch", "4",
                                  "--lidar", lidar, "--out", out]), log=lambda *a, **k: None)
        assert res["frames"] == len(KR.TRAIN)
        outs[lidar] = {f: open(os.path.join(out, f)).read() for f in sorted(os.listdir(out))}
    assert len(outs["velodyne"]) == len(KR.TRAIN) and outs["velodyne"] == outs["velodyne_reduced"]

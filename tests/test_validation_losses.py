"""Validating a checkpoint on a labelled split: the losses computed in the detection step itself (forward_points with
GT, the captured loss kind, detect_stream(losses=True), the driver's ``--losses``), the GT of KITTI labels
(kitti_data.gt_from_anno) and AP at 40 recall positions (kitti_eval.official_eval(recall_positions=40)).

CPU: gt_from_anno equals the reference's labelled test path bit for bit (tests/golden/gt_lidar.npz, made by
make_golden_gt.py) and Calibration.C2V its np.dot(-R.T, t); the R40 AP of the product and of the oracle's precision
arrays equals the AP of the reference's own eval_class_v3 arrays (tests/golden/eval_r40.npz, make_golden_eval_r40.py),
AOS included, and the R11 text is unchanged; the driver's arguments are checked; the gloo world-size-2 gather returns
every rank's per-batch loss vectors.
GPU: with GT the detections / KITTI rows are bit-identical to the same call without GT and the losses to loss_points,
eagerly, in the captured loss kind and in detect_stream at depth 4; 257 GT boxes raise on every path and the next
batch is right; the driver's ``--losses`` leaves the result files and AP untouched and its means are the means of
per-batch loss_points.
"""
import multiprocessing as mp
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist

from oracle import kitti_eval as O
from sassd_b200 import kitti_data as K
from sassd_b200 import kitti_eval as KE
from sassd_b200.results import Calibration

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLASS_LISTS = (["Car"], ["Car", "Pedestrian", "Cyclist"])
EVAL_KEYS = ('name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location', 'rotation_y')


# ------------------------------------------------------------------------------------------------------------ CPU
def test_gt_from_anno_equals_the_reference_labelled_test_path(golden_dir):
    g = np.load(os.path.join(golden_dir, "gt_lidar.npz"))
    ncalib = int(g["ncalib"])
    with tempfile.TemporaryDirectory() as d:
        calibs = []
        for c in range(ncalib):
            path = os.path.join(d, "calib%d.txt" % c)
            with open(path, "w") as fh:
                fh.write(str(g["calib_txt_%d" % c]))
            calibs.append(Calibration(path))
            assert np.array_equal(calibs[c].C2V, g["c2v_%d" % c]), c       # bit for bit, not just close
        n_boxes = 0
        for i in range(int(g["nframes"])):
            path = os.path.join(d, "%06d.txt" % i)
            with open(path, "w") as fh:
                fh.write(str(g["label_txt_%d" % i]))
            anno = K.read_label(path)
            for ci, names in enumerate(CLASS_LISTS):
                boxes, labels = K.gt_from_anno(anno, calibs[i % ncalib], names)
                assert boxes.dtype == np.float32 and boxes.shape[1:] == (7,) and labels.dtype == np.int64
                key = "%d_%d" % (ci, i)
                if int(g["error_" + key]):          # only DontCare rows: the reference fails, we give no GT
                    assert boxes.shape == (0, 7) and labels.shape == (0,)
                    continue
                np.testing.assert_array_equal(boxes, g["boxes_" + key])
                np.testing.assert_array_equal(labels, g["labels_" + key])
                n_boxes += len(boxes)
    assert n_boxes > 10


def _eval_annos(golden_dir):
    g = np.load(os.path.join(golden_dir, "eval.npz"))
    n = int(g['nframes'])
    gts = [{k: g['gt%d_%s' % (i, k)] for k in EVAL_KEYS} for i in range(n)]
    dts = [{k: g['dt%d_%s' % (i, k)] for k in EVAL_KEYS + ('score',)} for i in range(n)]
    return g, gts, dts


def _r40(prec):
    """AP over recall positions 1/40 ... 1 of the 41 samples, summed in sample order."""
    s = 0
    for i in range(1, 41):
        s = s + prec[..., i]
    return s / 40 * 100


def test_r40_ap_equals_the_reference_precision_arrays(golden_dir):
    g, gts, dts = _eval_annos(golden_dir)
    r = np.load(os.path.join(golden_dir, "eval_r40.npz"))
    want = dict(bbox=_r40(r["prec_0"]), bev=_r40(r["prec_1"]), d3=_r40(r["prec_2"]), aos=_r40(r["orient_0"]))
    text, ap = KE.official_eval(gts, dts, [0, 1, 2], overlap_fn=O.rotate_iou_eval, recall_positions=40)
    for k, v in want.items():
        np.testing.assert_array_equal(ap[k], v, err_msg=k)
    assert "Car AP_R40@0.70, 0.70, 0.70:" in text and text.count("AP_R40@") == 6
    # the oracle's precision arrays give the same AP
    overlaps = np.stack([KE.OVERLAP_0_7, KE.OVERLAP_0_5], 0)[:, :, [0, 1, 2]]
    for metric, key in ((0, "bbox"), (1, "bev"), (2, "d3")):
        o = O.eval_classes(gts, dts, [0, 1, 2], [0, 1, 2], metric, overlaps, compute_aos=metric == 0)
        np.testing.assert_array_equal(_r40(o["precision"]), want[key], err_msg=key)
        if metric == 0:
            np.testing.assert_array_equal(_r40(o["orientation"]), want["aos"])
    # R11 is untouched: the reference's text and APs, by default and when asked for
    for kw in ({}, {"recall_positions": 11}):
        text11, ap11 = KE.official_eval(gts, dts, [0, 1, 2], overlap_fn=O.rotate_iou_eval, **kw)
        assert text11 == str(g["official_text"])
        np.testing.assert_array_equal(ap11["d3"], g["ap_d3"])
    with pytest.raises(ValueError, match="11 or 40"):
        KE.official_eval(gts, dts, [0], overlap_fn=O.rotate_iou_eval, recall_positions=41)


def test_driver_arguments():
    from sassd_b200 import test as T
    cfg = os.path.join(ROOT, "configs", "car_cfg.py")
    for bad in (["--drive", "d", "--out", "o", "--losses"], ["--data-root", "r", "--split", "test", "--out", "o",
                                                              "--losses"],
                ["--drive", "d", "--out", "o", "--r40"], ["--data-root", "r", "--split", "test", "--out", "o", "--r40"]):
        with pytest.raises(SystemExit):
            T.parse_args([cfg, "w.pth"] + bad)
    a = T.parse_args([cfg, "w.pth", "--data-root", "r", "--losses", "--r40"])
    assert a.losses and a.r40 and a.split == "val"
    a = T.parse_args([cfg, "w.pth", "--data-root", "r"])
    assert not a.losses and not a.r40


def _label_line(name, rng):
    vals = [0.0, 0, round(float(rng.uniform(-3, 3)), 2)] + [100.0, 150.0, 200.0, 220.0]
    vals += [1.5, 1.6, 3.9, round(float(rng.uniform(-10, 10)), 2), 1.7, round(float(rng.uniform(5, 50)), 2),
             round(float(rng.uniform(-3, 3)), 2)]
    return " ".join([name] + [str(v) for v in vals])


def test_split_yields_the_ground_truth_with_each_batch(tmp_path, golden_dir):
    from tests.test_kitti_data import write_split
    g = np.load(os.path.join(golden_dir, "results.npz"))
    ids = [4, 9, 11]
    write_split(str(tmp_path), ids, [(375, 1242)], [str(g["calib_txt"])], [np.ones((3, 4)) * k for k in range(3)])
    rng = np.random.default_rng(0)
    rows = {4: ["Car", "Van", "DontCare"], 9: ["Pedestrian"], 11: []}
    for i, names in rows.items():
        with open(os.path.join(str(tmp_path), "training", "label_2", "%06d.txt" % i), "w") as fh:
            fh.write("".join(_label_line(n, rng) + "\n" for n in names))
    split = K.KittiSplit(str(tmp_path), "val", "velodyne_reduced", gt_classes=["Car"])
    got = list(K.Prefetcher(split, K.padded_batches(ids, 2), depth=1, workers=2))
    assert [b[0] for b in got] == [[4, 9], [11, None]]
    gts = [gt for b in got for gt in b[3]]
    assert [len(b) for b, _ in gts] == [2, 0, 0, 0]           # Van counts as Car; padding has no GT
    calib = split.meta(4)["calib"]
    want = K.gt_from_anno(K.read_label(split.path("label_2", 4, "txt")), calib, ["Car"])
    assert np.array_equal(gts[0][0], want[0]) and gts[0][1].tolist() == [1, 1]
    # without gt_classes the batches are as before
    assert all(len(b) == 3 for b in K.Prefetcher(K.KittiSplit(str(tmp_path), "val"), [[4, 9]], workers=1))
    with open(os.path.join(str(tmp_path), "ImageSets", "test.txt"), "w") as fh:
        fh.write("000004\n")
    with pytest.raises(ValueError, match="no labels"):
        K.KittiSplit(str(tmp_path), "test", gt_classes=["Car"])


def test_loss_kind_keys_and_threshold_check():
    import sassd_b200 as S
    model, _, _ = S.build_from_config(S.Config.fromfile(os.path.join(ROOT, "configs", "car_cfg.py")), device="cpu")
    model._require_loss_step()              # both shipped configs select the guided anchors at the test threshold
    # the loss kind has a four-element key; the other kinds keep theirs, so (False, False, False) still names the plain
    # kind (the graphs are disabled: _graph_for only looks up)
    model._graphs = {(False, False, False): "plain", (0, False, False, True): "losses"}
    assert model._graph_for(0, False, False) == "plain" and model._graph_for(0, False, False, True) == "losses"
    assert model._graph_for(1, False, False, True) is None
    model.refresh_packed_weights()
    assert model._graphs == {}
    model.train_cfg.rpn.anchor_thr = 0.2
    with pytest.raises(ValueError, match="anchor_thr"):
        model._require_loss_step()


def _gather_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    from sassd_b200 import dist as D
    from sassd_b200.test import gather_losses
    D.init_from_env(backend="gloo")
    # three batches per rank; rank 1's last batch is all padding
    local = [[rank * 10 + j + k / 8.0 for k in range(6)] for j in range(3)]
    n_real = [2, 2, 1] if rank == 0 else [2, 1, 0]
    q.put((rank, gather_losses(local, n_real, torch.device("cpu"))))
    dist.destroy_process_group()


def test_loss_gather_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    vec = lambda r, j: [np.float32(r * 10 + j + k / 8.0).item() for k in range(6)]     # noqa: E731
    want = [vec(0, 0), vec(1, 0), vec(0, 1), vec(1, 1), vec(0, 2)]      # (batch, rank) order, padding batch dropped
    for _, got in res:
        assert got == want


# ------------------------------------------------------------------------------------------------------------ GPU
def _same_results(got, want):
    """Detection dicts or KITTI annotation dicts, bit for bit."""
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert set(g) == set(w)
        for k in w:
            if w[k] is None or g[k] is None:
                assert g[k] is None and w[k] is None, k
            else:
                assert np.asarray(g[k]).dtype == np.asarray(w[k]).dtype and np.array_equal(g[k], w[k]), k


def _inputs(golden_dir, B, nc, seed0=0):
    """B frames: cropped-size clouds (about 20 k points) for the uncropped kind, full sweeps with their metas and
    frustum planes for the cropping kinds, and GT cars (frame 1 without GT)."""
    from sassd_b200.synth import synth_cloud
    from tests.test_kitti_format import _sweeps_and_metas
    from tests.test_losses import _frames
    seeds = [seed0 + b for b in range(B)]
    full, metas, planes = _sweeps_and_metas(golden_dir, seeds)
    _, gts, labels = _frames(B, nc, empty=(1,))
    return dict(small=[synth_cloud(s) for s in seeds], full=full, metas=metas, planes=planes, gts=gts, labels=labels)


KINDS = ("plain", "crop_kitti", "crop")
MAX_POINTS = dict(plain=32768, crop_kitti=131072, crop=131072)


def _kw(kind, f):
    """forward_points' points and arguments of a kind."""
    if kind == "plain":
        return f["small"], {}
    kw = dict(frustum_planes=f["planes"])
    if kind == "crop_kitti":
        kw["metas"] = f["metas"]
    return f["full"], kw


def _release(model):
    """Drop every captured step and return its memory (a batch of 16 full sweeps captures several GB per step)."""
    import gc
    model.disable_cuda_graph()
    model.refresh_packed_weights()
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name", ["car_cfg.py", "multi_cfg.py"])
def test_loss_step_eager_captured_and_streamed(golden_dir, cfg_name):
    """Eager: every kind at B = 1, 2, 16.  Captured: every loss kind at B = 1, 2, the uncropped one at 16.  Streamed
    (depth 4, concurrent slots): the uncropped kind at every B, the crop + KITTI kind at B = 1, 2."""
    from tests.test_losses import _model
    model = _model(cfg_name)
    nc = len(model.class_names)
    nonzero = 0
    for B in (1, 2, 16):
        batches = [_inputs(golden_dir, B, nc, seed0=100 * s) for s in range(5 if B < 16 else 2)]
        kinds = KINDS if B < 16 else ("plain",)
        want = {}
        for kind in KINDS:
            for s, f in enumerate(batches):
                pts, kw = _kw(kind, f)
                res, losses = model.forward_points(pts, gt_bboxes=f["gts"], gt_labels=f["labels"], **kw)
                _same_results(res, model.forward_points(pts, **kw))
                assert losses == model.loss_points(pts, f["gts"], f["labels"], frustum_planes=kw.get("frustum_planes"))
                nonzero += sum(v != 0 for v in losses.values())
                want[kind, s] = (res, losses)
        # the captured loss kinds
        model.enable_cuda_graph(B, 131072 if B < 16 else 32768)
        for kind in kinds:
            pts, kw = _kw(kind, batches[0])
            res, losses = model.forward_points(pts, gt_bboxes=batches[0]["gts"], gt_labels=batches[0]["labels"], **kw)
            _same_results(res, want[kind, 0][0])
            assert losses == want[kind, 0][1], (kind, B)
        assert {k for k in model._graphs if len(k) == 4} == {
            dict(plain=(0, False, False, True), crop_kitti=(1, True, False, True), crop=(1, False, False, True))[k]
            for k in kinds}
        _release(model)
        # streamed, depth 4, concurrent slots
        for kind in kinds[:2]:
            if kind == "plain":
                items = [(f["small"], (f["gts"], f["labels"])) for f in batches]
            else:
                items = [(f["full"], f["planes"], f["metas"], (f["gts"], f["labels"])) for f in batches]
            got = list(model.detect_stream(items, B, MAX_POINTS[kind], depth=4, crop=kind != "plain",
                                           kitti=kind == "crop_kitti", losses=True))
            assert len(got) == len(batches)
            for s, (res, losses) in enumerate(got):
                _same_results(res, want[kind, s][0])
                assert losses == want[kind, s][1], (kind, B, s)
            _release(model)
    assert nonzero > 20


@pytest.mark.gpu
def test_gt_capacity_overflow_raises_on_every_path_and_the_next_batch_is_right(golden_dir):
    from sassd_b200.lib import GT_CAP_MAX, SassdError
    from tests.test_losses import _model
    model = _model()
    f = _inputs(golden_dir, 2, 1)
    pts, gts, labels = f["small"], f["gts"], f["labels"]
    many = np.repeat(gts[0][:1], GT_CAP_MAX + 1, 0)
    bad = dict(gt_bboxes=[many, gts[1]], gt_labels=[np.ones(len(many), np.int64), labels[1]])
    res_want, loss_want = model.forward_points(pts, gt_bboxes=gts, gt_labels=labels)
    with pytest.raises(SassdError, match="GT_CAP"):
        model.forward_points(pts, **bad)
    model.enable_cuda_graph(2, 32768)
    for _ in range(2):
        with pytest.raises(SassdError, match="GT_CAP"):
            model.forward_points(pts, **bad)
        res, losses = model.forward_points(pts, gt_bboxes=gts, gt_labels=labels)
        _same_results(res, res_want)
        assert losses == loss_want
    items = [(pts, (bad["gt_bboxes"], bad["gt_labels"])), (pts, (gts, labels))]
    with pytest.raises(SassdError, match="GT_CAP"):
        list(model.detect_stream(items, 2, 32768, depth=4, losses=True))
    (res, losses), = list(model.detect_stream(items[1:], 2, 32768, depth=4, losses=True))
    _same_results(res, res_want)
    assert losses == loss_want


@pytest.mark.gpu
def test_driver_losses_leave_the_results_and_ap_untouched(golden_dir, tmp_path):
    import sassd_b200 as S
    from sassd_b200 import checkpoint, ops
    from sassd_b200 import test as T
    from sassd_b200.frustum import camera_frustum_planes
    from sassd_b200.results import annos_to_kitti_label, kitti_bbox2results
    from sassd_b200.synth import synth_cloud
    from tests.test_kitti_data import write_split
    from tests.test_kitti_format import _calib_txt, _calibs
    from tests.test_point_aux import _aux_weights
    rng = np.random.default_rng(9)
    ids = [int(i) for i in np.sort(rng.choice(7000, 11, replace=False))]
    calibs = _calibs(golden_dir)
    root = str(tmp_path / "kitti")
    write_split(root, ids, [(375, 1242), (370, 1224)], [_calib_txt(c) for c in calibs],
                [synth_cloud(2000 + j, fov_deg=180.0) for j in range(len(ids))])
    sd = checkpoint.make_synthetic_state_dict(0, 1)
    sd.update(_aux_weights())
    ckpt = str(tmp_path / "synthetic.pth")
    checkpoint.save_checkpoint(sd, ckpt)
    split = K.KittiSplit(root, "val", "velodyne")
    for j, i in enumerate(ids):            # labels: cars near the synthetic ones, a Van, DontCare rows, one empty frame
        m = split.meta(i)
        n = 0 if j == 3 else int(rng.integers(1, 6))
        boxes = np.stack([rng.uniform(8, 40, n), rng.uniform(-6, 6, n), np.full(n, -1.7), np.full(n, 1.6),
                          np.full(n, 3.9), np.full(n, 1.56), rng.uniform(-3, 3, n)], 1).astype(np.float32)
        gt = kitti_bbox2results(boxes.copy(), np.ones(n, np.float32), np.zeros(n, np.int64), m, ["Car"])
        gt = dict(gt, dimensions=gt["dimensions"][:, [1, 2, 0]])
        lines = annos_to_kitti_label(gt)
        if n > 1:
            lines[1] = "Van" + lines[1][3:]
        if j % 2:       # the written lines carry a score field; a DontCare line among them must too
            lines.append(_label_line("DontCare", rng) + (" 1.0" if lines else ""))
        with open(os.path.join(root, "training", "label_2", "%06d.txt" % i), "w") as fh:
            fh.write("".join(l + "\n" for l in lines))

    cfg = os.path.join(ROOT, "configs", "car_cfg.py")
    B = 4
    base = ["--data-root", root, "--batch", str(B), "--workers", "2"]
    out0, out1 = str(tmp_path / "plain"), str(tmp_path / "losses")
    printed = []
    r0 = T.run(T.parse_args([cfg, ckpt, "--out", out0] + base), log=lambda *a, **k: None)
    import gc
    gc.collect()
    torch.cuda.empty_cache()            # each run builds its own model and captured slots
    r1 = T.run(T.parse_args([cfg, ckpt, "--out", out1, "--losses", "--r40"] + base),
               log=lambda *a, **k: printed.append(" ".join(a)))
    files = lambda d: {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d))}     # noqa: E731
    assert files(out0) == files(out1) and len(files(out0)) == len(ids)
    assert r1["text"] == r0["text"] and r1["ap"] == r0["ap"] and printed[0] == r0["text"]
    assert "ap_r40" in r1 and "AP_R40@" in r1["text_r40"] and printed[1] == r1["text_r40"]
    # the losses: per-batch loss_points on the driver's batches (the last one padded with empty frames)
    model, _, _ = S.build_from_config(S.Config.fromfile(cfg), device="cuda:0")
    checkpoint.load_params_from_file(model, ckpt)
    gsplit = K.KittiSplit(root, "val", "velodyne", gt_classes=["Car"])
    per_batch = []
    for ids_b in K.padded_batches(ids, B):
        frames = [gsplit.frame(i) if i is not None else gsplit.pad_frame() for i in ids_b]
        losses = model.loss_points([p for p, _, _ in frames], [g[0] for _, _, g in frames],
                                   [g[1] for _, _, g in frames], frustum_planes=[
                                       camera_frustum_planes(m["calib"], m["img_shape"]) for _, m, _ in frames])
        per_batch.append([losses[k] for k in ops.LOSS_KEYS])
    assert [[d[k] for k in ops.LOSS_KEYS] for d in r1["losses_per_batch"]] == per_batch
    means = np.mean(np.asarray(per_batch, np.float64), axis=0)
    assert [r1["losses"][k] for k in ops.LOSS_KEYS] == means.tolist()
    assert any(v > 0 for v in means) and "mean over 3 batches" in printed[2]

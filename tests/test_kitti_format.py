"""KITTI result formatting on the device (csrc/kitti_format.cu, ops.kitti_format, forward_points(metas=),
detect_stream(kitti=True)) and the split evaluation driver (python -m sassd_b200.test).

The device formatter follows results.kitti_bbox2results dtype by dtype but not bit for bit: numpy's float32
sin / cos / atan2, its einsum and OpenBLAS's dgemm summation order are not CUDA's.  The bounds, per field:
  * name, label, score, dimensions: copies of the fp32 detection -> equal;
  * rotation_y: the fp32 yaw wrap is the same sequence of correctly rounded operations -> within 1 fp32 ulp;
  * location: an fp64 product of an fp32 point, rounded to fp32; a different fp64 summation order moves the fp64 value
    by ~1e-16 relative, which can only flip the final fp32 rounding -> within 1 fp32 ulp;
  * alpha: -atan2f(-y, x) + ry in fp32; the atan2 implementations differ by a few ulp of a value below pi
    (2.4e-7 each) and the sum is rounded once more -> within 1e-6 rad;
  * bbox: fp64 projection of fp32 corners whose sin / cos / products differ by about an fp32 ulp (6e-8 relative) of
    metre-scale coordinates; at KITTI's focal length (721 px) that is 1e-5 to 1e-4 px for boxes a few metres from
    the camera, more only for corners close to the image plane -> 1e-3 px.
A keep decision can only differ for a box whose host bbox lies within those 1e-3 px of an image edge."""
import os

import numpy as np
import pytest
import torch

from sassd_b200.results import (Calibration, annos_from_rows, camera_box_corners, kitti_bbox2results, limit_period,
                                meta_block, project_rect_to_image, project_velo_to_rect)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["Car", "Pedestrian", "Cyclist"]
SHAPES = [(375, 1242, 3), (370, 1224, 3), (376, 1241, 3)]
BBOX_TOL, ALPHA_TOL = 1e-3, 1e-6


def _ulp_close(a, b, what):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert np.all(np.abs(a.astype(np.float64) - b) <= np.spacing(np.abs(b))), (what, a, b)


def same_annos(dev, host, what=""):
    """Field-by-field bounds of the module docstring, for one frame kept identically."""
    assert len(dev["name"]) == len(host["name"]), (what, len(dev["name"]), len(host["name"]))
    assert set(dev) == set(host), what
    if len(host["name"]) == 0:
        return 0
    for k in ("name", "truncated", "occluded", "image_idx"):
        assert np.array_equal(dev[k], host[k]), (what, k)
    for k in ("score", "dimensions"):
        assert dev[k].dtype == host[k].dtype and np.array_equal(dev[k], host[k]), (what, k)
    for k in ("alpha", "location", "rotation_y", "bbox"):
        assert dev[k].dtype == host[k].dtype, (what, k)
    _ulp_close(dev["location"], host["location"], what + " location")
    _ulp_close(dev["rotation_y"], host["rotation_y"], what + " rotation_y")
    assert np.abs(dev["alpha"].astype(np.float64) - host["alpha"]).max() <= ALPHA_TOL, what
    assert np.abs(dev["bbox"] - host["bbox"]).max() <= BBOX_TOL, what
    return len(host["name"])


def _format_on_device(dets, metas, cap):
    """dets: per frame [n,9] f32 (x,y,z,w,l,h,ry,score,label) -> device annos."""
    from sassd_b200 import ops
    B = len(dets)
    det = np.zeros((B, cap, 9), np.float32)
    nd = np.zeros(B, np.int32)
    for b, d in enumerate(dets):
        det[b, :len(d)] = d
        nd[b] = len(d)
    dev = torch.device("cuda:0")
    meta = torch.from_numpy(np.stack([meta_block(m["calib"], m["img_shape"]) for m in metas])).to(dev)
    rows, n_out = ops.kitti_format(torch.from_numpy(det).to(dev), torch.from_numpy(nd).to(dev), meta)
    torch.cuda.synchronize()
    return annos_from_rows(rows.cpu().numpy(), n_out.cpu().numpy(), NAMES, [m["sample_idx"] for m in metas])


def _host(d, meta):
    return kitti_bbox2results(d[:, :7].copy(), d[:, 7].copy(), d[:, 8].astype(np.int64), meta, NAMES)


# ------------------------------------------------------------------ 1. the reference's own outputs
@pytest.mark.gpu
def test_against_the_reference_outputs(golden_dir, tmp_path):
    g = np.load(os.path.join(golden_dir, "results.npz"))
    p = tmp_path / "calib.txt"
    p.write_text(str(g["calib_txt"]))
    calib = Calibration(str(p))
    dets, metas, wants = [], [], []
    for ci in range(int(g["ncases"])):
        b = g["c%d_boxes" % ci]
        dets.append(np.concatenate([b, g["c%d_scores" % ci][:, None], g["c%d_labels" % ci][:, None]], 1)
                    .astype(np.float32))
        metas.append(dict(calib=calib, sample_idx=100 + ci, img_shape=(375, 1242, 3)))
        wants.append({k[len("c%d_out_" % ci):]: g[k] for k in g.files if k.startswith("c%d_out_" % ci)})
    got = _format_on_device(dets, metas, 512)
    n = sum(same_annos(d, w, "case %d" % i) for i, (d, w) in enumerate(zip(got, wants)))
    assert n > 10


# ------------------------------------------------------------------ 2. randomised batches
def _calibs(golden_dir):
    z = np.load(os.path.join(golden_dir, "frustum.npz"))
    return [Calibration({"P2": z["calib%d_P2" % c], "Tr_velo_to_cam": z["calib%d_Tr" % c],
                         "R0_rect": z["calib%d_R0" % c]}) for c in range(2)]


def _random_dets(rng, n, frame):
    """Boxes inside the image, straddling its left / right edge, wholly outside it (beside or behind the camera);
    yaws uniform and around +-pi, +-2pi.  Scores are distinct so that rows can be matched to boxes."""
    kind = rng.integers(0, 4, n)
    x = np.where(kind == 3, rng.uniform(-40, -4, n), rng.uniform(4, 70, n))
    edge = x * 0.86                                        # |y| of the left / right image edge at depth x
    y = np.select([kind == 0, kind == 1, kind == 2],
                  [rng.uniform(-0.6, 0.6, n) * edge, np.sign(rng.normal(size=n)) * (edge + rng.uniform(-2, 2, n)),
                   np.sign(rng.normal(size=n)) * (1.5 * edge + 6)], rng.uniform(-30, 30, n))
    yaw = np.where(rng.random(n) < 0.5, rng.uniform(-8, 8, n),
                   rng.choice([-2 * np.pi, -np.pi, np.pi, 2 * np.pi], n) + rng.normal(0, 1e-3, n))
    d = np.stack([x, y, rng.uniform(-2.5, 0, n), rng.uniform(0.5, 2.2, n), rng.uniform(0.6, 5, n),
                  rng.uniform(1.2, 2, n), yaw, np.zeros(n), rng.integers(0, 3, n)], 1).astype(np.float32)
    d[:, 7] = (frame * 4096 + rng.permutation(n) + 1) / np.float32(1 << 22)
    return d


def _host_decisions(d, meta):
    """The host formatter's keep decision per box, and whether its bbox lies within BBOX_TOL of an image edge."""
    calib, (h, w) = meta["calib"], meta["img_shape"][:2]
    b = d[:, :7].copy()
    b[:, 6] = limit_period(b[:, 6], offset=0.5, period=np.pi * 2)
    cam = np.zeros_like(b)
    cam[:, :3] = project_velo_to_rect(b[:, :3], calib)
    cam[:, 3:] = b[:, [4, 5, 3, 6]]
    img = project_rect_to_image(camera_box_corners(cam), calib)
    box = np.concatenate([img.min(1), img.max(1)], 1)
    keep = ~((box[:, 0] > w) | (box[:, 1] > h) | (box[:, 2] < 0) | (box[:, 3] < 0))
    near = (np.abs(box[:, 0] - w) <= BBOX_TOL) | (np.abs(box[:, 1] - h) <= BBOX_TOL) | \
        (np.abs(box[:, 2]) <= BBOX_TOL) | (np.abs(box[:, 3]) <= BBOX_TOL)
    return keep, near


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2, 16])
def test_randomised_batches_match_the_host_formatter(golden_dir, B):
    rng = np.random.default_rng(B)
    calibs, cap = _calibs(golden_dir), 512
    sizes = {1: [cap], 2: [0, 1]}.get(B, [0, 1, cap] + list(rng.integers(2, cap, 13)))
    dets = [_random_dets(rng, int(n), b) for b, n in enumerate(sizes)]
    metas = [dict(calib=calibs[b % 2], img_shape=SHAPES[b % 3], sample_idx=7 * b) for b in range(B)]
    got = _format_on_device(dets, metas, cap)
    n_kept, n_near, n_flip = 0, 0, 0
    for b, (d, m, dev) in enumerate(zip(dets, metas, got)):
        host = _host(d, m)
        keep, near = _host_decisions(d, m)
        assert int(keep.sum()) == len(host["name"])
        if len(d):
            n_near += int(near.sum())
        pos = {float(s): i for i, s in enumerate(d[:, 7])}
        dev_keep = np.zeros(len(d), bool)
        dev_keep[[pos[float(s)] for s in dev["score"]]] = True
        flip = dev_keep != keep
        assert not (flip & ~near).any(), "frame %d: keep decisions differ away from the image edge" % b
        n_flip += int(flip.sum())
        if flip.any():              # compare the boxes both kept
            both = keep & dev_keep
            if not both.any():
                continue
            host = _host(d[both], m)
            sel = np.isin(dev["score"], d[both, 7])
            dev = {k: v[sel] for k, v in dev.items()}
        n_kept += same_annos(dev, host, "B=%d frame %d" % (B, b))
    print("B=%d: %d rows compared, %d boxes within %g px of an edge, %d keep decisions differ"
          % (B, n_kept, n_near, BBOX_TOL, n_flip))
    if B != 2:
        assert n_kept > 0


# ------------------------------------------------------------------ 3. through the step
def _model():
    import sassd_b200 as S
    from sassd_b200 import checkpoint
    cfg = S.Config.fromfile(os.path.join(ROOT, "configs", "car_cfg.py"))
    model, _, _ = S.build_from_config(cfg, device="cuda:0")
    checkpoint.load_state_dict_into(model, checkpoint.make_synthetic_state_dict(0, 1))
    return model


def _sweeps_and_metas(golden_dir, seeds):
    from sassd_b200.frustum import camera_frustum_planes
    from sassd_b200.synth import synth_cloud
    calibs = _calibs(golden_dir)
    pts = [synth_cloud(s, fov_deg=180.0) for s in seeds]
    metas = [dict(calib=calibs[j % 2], img_shape=SHAPES[j % 3], sample_idx=s) for j, s in enumerate(seeds)]
    planes = [camera_frustum_planes(m["calib"], m["img_shape"]) for m in metas]
    return pts, metas, planes


def _host_of(dets, metas):
    out = []
    for d, m in zip(dets, metas):
        if d["boxes_lidar"] is None:
            out.append(kitti_bbox2results(None, None, None, m, NAMES))
        else:
            out.append(kitti_bbox2results(d["boxes_lidar"].copy(), d["scores"], d["label_preds"], m, NAMES))
    return out


@pytest.mark.gpu
def test_forward_points_and_detect_stream_format_like_the_host(golden_dir):
    from sassd_b200.single_stage_heads import unpack_detections
    model = _model()
    model.class_names = NAMES
    pts, metas, planes = _sweeps_and_metas(golden_dir, [0, 1, 2, 3])
    n = 0
    # eager, on reduced-range clouds and on full sweeps cropped on the device
    for kw in ({}, dict(frustum_planes=planes[:2])):
        got, aux = model.forward_points(pts[:2], metas=metas[:2], return_aux=True, **kw)
        bbs, scs, lbs = unpack_detections(aux["det"], aux["ndet"])
        dets = [dict(boxes_lidar=b, scores=s, label_preds=l) for b, s, l in zip(bbs, scs, lbs)]
        n += sum(same_annos(g, h, "eager %s" % list(kw)) for g, h in zip(got, _host_of(dets, metas[:2])))
    assert n > 0, "no detection to compare"
    # captured: the formatting graphs against host formatting of the plain graphs' detections
    model.enable_cuda_graph(2, 131072)
    for kw in ({}, dict(frustum_planes=planes[2:])):
        plain = model.forward_points(pts[2:], **kw)
        got = model.forward_points(pts[2:], metas=metas[2:], **kw)
        n += sum(same_annos(g, h, "graph %s" % list(kw)) for g, h in zip(got, _host_of(plain, metas[2:])))
    assert set(model._kitti_graphs) == {False, True}
    model.disable_cuda_graph()
    # detect_stream: formatting crop slots against plain crop slots + host formatting
    order = [(0, 1), (2, 3), (1, 2)]
    got = list(model.detect_stream([([pts[i] for i in o], [planes[i] for i in o], [metas[i] for i in o])
                                    for o in order], 2, 131072, depth=2, crop=True, kitti=True))
    plain = list(model.detect_stream([([pts[i] for i in o], [planes[i] for i in o]) for o in order], 2, 131072,
                                     depth=2, crop=True))
    assert len(got) == len(plain) == len(order)
    for o, g, p in zip(order, got, plain):
        for gi, hi in zip(g, _host_of(p, [metas[i] for i in o])):
            n += same_annos(gi, hi, "stream")
    with pytest.raises(ValueError):
        model.class_names = None
        model.forward_points(pts[:1], metas=metas[:1])


# ------------------------------------------------------------------ 4. the driver end to end
def _calib_txt(c):
    fmt = lambda a: " ".join("%.12e" % v for v in np.asarray(a).ravel())      # noqa: E731
    return "P2: %s\nR0_rect: %s\nTr_velo_to_cam: %s\n" % (fmt(c.P2), fmt(c.R0), fmt(c.V2C))


@pytest.mark.gpu
def test_driver_end_to_end(golden_dir, tmp_path):
    from sassd_b200 import checkpoint, kitti_data as K
    from sassd_b200 import test as T
    from sassd_b200.frustum import camera_frustum_planes
    from sassd_b200.kitti_eval import official_eval
    from sassd_b200.results import annos_to_kitti_label
    from sassd_b200.synth import synth_cloud
    from tests.test_kitti_data import write_split
    rng = np.random.default_rng(5)
    ids = [int(i) for i in np.sort(rng.choice(7000, 37, replace=False))]
    calibs = _calibs(golden_dir)
    shapes = [(375, 1242), (370, 1224)]
    pts = [synth_cloud(1000 + j, fov_deg=180.0) for j in range(len(ids))]
    root = str(tmp_path / "kitti")
    write_split(root, ids, shapes, [_calib_txt(c) for c in calibs], pts)
    ckpt = str(tmp_path / "synthetic.pth")
    checkpoint.save_checkpoint(checkpoint.make_synthetic_state_dict(0, 1), ckpt)

    # the composition the driver must equal: forward_points on full sweeps + host formatting + evaluation
    model = _model()
    split = K.KittiSplit(root, "val", "velodyne")
    frames = [split.frame(i) for i in ids]
    assert [m["img_shape"][:2] for _, m in frames[:2]] == shapes
    dets = []
    for s in range(0, len(ids), 16):
        chunk = frames[s:s + 16]
        dets += model.forward_points([p for p, _ in chunk], frustum_planes=[
            camera_frustum_planes(m["calib"], m["img_shape"]) for _, m in chunk])
    dt = [kitti_bbox2results(None if d["boxes_lidar"] is None else d["boxes_lidar"].copy(), d["scores"],
                             d["label_preds"], m, ["Car"]) for d, (_, m) in zip(dets, frames)]
    # ground truth: the detections' lidar boxes jittered, a few removed, a few cars added
    n_det = 0
    for j, (d, (_, m)) in enumerate(zip(dets, frames)):
        boxes = np.zeros((0, 7), np.float32) if d["boxes_lidar"] is None else d["boxes_lidar"].copy()
        n_det += len(boxes)
        keep = rng.random(len(boxes)) > 0.15
        boxes = boxes[keep]
        boxes[:, :2] += rng.normal(0, 0.15, (len(boxes), 2)).astype(np.float32)
        boxes[:, 6] += rng.normal(0, 0.05, len(boxes)).astype(np.float32)
        if j % 5 == 0:
            extra = np.array([[rng.uniform(8, 40), rng.uniform(-5, 5), -1.0, 1.6, 3.9, 1.56, rng.uniform(-3, 3)]],
                             np.float32)
            boxes = np.concatenate([boxes, extra])
        gt = kitti_bbox2results(boxes.copy(), np.ones(len(boxes), np.float32), np.zeros(len(boxes), np.int64), m,
                                ["Car"])
        with open(os.path.join(root, "training", "label_2", "%06d.txt" % ids[j]), "w") as fh:
            gt = dict(gt, dimensions=gt["dimensions"][:, [1, 2, 0]])        # l, h, w -> the file's h, w, l
            fh.write("".join(line + "\n" for line in annos_to_kitti_label(gt)))
    assert n_det > 20
    gt_annos = split.gt_annos()
    text_want, ap_want = official_eval(gt_annos, dt, ["Car"])

    out, js = str(tmp_path / "results"), str(tmp_path / "ap.json")
    printed = []
    res = T.run(T.parse_args([os.path.join(ROOT, "configs", "car_cfg.py"), ckpt, "--data-root", root, "--batch", "16", "--out", out,
                              "--json", js, "--workers", "3"]), log=lambda *a, **k: printed.append(" ".join(a)))
    print(res["text"], "%.1f frames/s, read wait %.3f s" % (res["frames_per_s"], res["read_wait_s"]))
    assert res["frames"] == 37 and printed[0] == text_want and res["text"] == text_want
    # bbox / bev / 3d AP depend only on boxes, scores and keep decisions: equal.  AOS averages (1 + cos(d_alpha)) / 2
    # over the matches, and the device alpha differs from the host's by up to 1e-6 rad: equal to the table's 2
    # decimals, not bit for bit.
    for k in ("bbox", "bev", "d3"):
        assert np.array_equal(np.asarray(res["ap"][k]), ap_want[k]), k
    assert (ap_want["aos"] is None) == (res["ap"]["aos"] is None)
    if ap_want["aos"] is not None:
        assert np.abs(np.asarray(res["ap"]["aos"]) - ap_want["aos"]).max() <= 1e-6
    bbox3d = np.asarray(res["ap"]["d3"])
    assert 0 < bbox3d[0, 0, 0] < 100, bbox3d
    # result files parse back to the host annotations within the files' 4 decimals (5e-5) plus the device formatter's
    # bound of the field (module docstring; 1e-5 covers 1 fp32 ulp of coordinates below 128 m)
    back = K.read_labels(out, ids)
    tol = dict(alpha=ALPHA_TOL, bbox=BBOX_TOL, dimensions=0.0, location=1e-5, rotation_y=1e-5, score=0.0)
    for j, (b, d) in enumerate(zip(back, dt)):
        assert len(b["name"]) == len(d["name"]), j
        if len(d["name"]):
            for k, t in tol.items():
                assert np.abs(b[k] - d[k]).max() <= 5e-5 + t + 1e-9, (j, k)
    assert sorted(os.listdir(out)) == ["%06d.txt" % i for i in ids]


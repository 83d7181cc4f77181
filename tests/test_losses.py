"""SA-SSD's training targets and losses, forward only (csrc/targets.cu, SingleStageDetector.forward_train /
loss_points).

CPU: the numpy restatement (oracle/targets.py) equals the reference's own pts_in_boxes3d (points_op.cpp, built
unmodified by __graft_entry__.build() into oracle/_ref/) and hand-derived assignments; training mode still raises.
GPU: point flags and offsets, RPN labels and max IoUs are bit-identical to the oracle (and the built reference
extension); box targets within 2 ulp; every loss within rel 1e-5 of the oracle on the same inputs; forward(return_loss=
True) equals loss_points; repeated calls give the same bits; detections are unchanged by a loss call; frames without
GT, multi_cfg and the GT capacity are covered.
Golden (tests/golden/loss.npz, made by make_golden_loss.py from the reference's own create_target_torch,
SSDRotateHead.loss, PSWarpHead.loss and SpMiddleFHD.aux_loss): the oracle reproduces it on the CPU (labels and flags
exact, targets within 1e-6, losses within rel 1e-6) and the kernels reproduce it on the GPU (labels, flags and offsets
exact, targets within 2 ulp, losses within rel 1e-5).  PSWarp's IoUs are also held bit for bit to the reference's
boxesoverlapLauncher when build() made it.
"""
import os

import numpy as np
import pytest
import torch

from oracle import targets as OT
from tests.test_point_aux import _aux_weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def _ref_ext():
    from oracle import points_op_ref
    return points_op_ref.load()


def _constructed_points_and_boxes(seed=0):
    """Boxes that overlap and touch, points on their faces, corners and inside two boxes, plus random points."""
    rng = np.random.default_rng(seed)
    boxes = np.array([[10.0, 2.0, -1.7, 1.6, 3.9, 1.56, 0.0],
                      [11.0, 2.5, -1.7, 1.6, 3.9, 1.56, 0.3],          # overlaps box 0
                      [20.0, -5.0, -1.5, 0.6, 0.8, 1.7, np.pi / 2],
                      [30.0, 8.0, -1.6, 2.0, 4.5, 1.8, -2.9]], f32)
    pts = [rng.uniform([5, -10, -3], [35, 12, 1], (4000, 3))]
    for b in boxes:
        c, s = np.cos(b[6]), np.sin(b[6])
        for u in (-0.5, 0.0, 0.5):
            for v in (-0.5, 0.0, 0.5):
                lx, ly = u * b[3], v * b[4]
                pts.append(np.array([[b[0] + lx * c - ly * s, b[1] + lx * s + ly * c, b[2] + b[5] * t]
                                     for t in (0.0, 0.5, 1.0)]))
        pts.append(b[None, :3] + rng.normal(0, 0.5, (300, 3)) * [b[3], b[4], b[5]])
    pts.append(np.array([[10.5, 2.25, -1.0]]))                       # inside boxes 0 and 1
    return np.ascontiguousarray(np.concatenate(pts).astype(f32)), boxes


# ------------------------------------------------------------------------------------------------------------ CPU
def test_oracle_pts_in_boxes3d_equals_the_reference_extension():
    ext = _ref_ext()
    if ext is None:
        pytest.skip("the reference points_op extension was not built (no checkout of the original project)")
    for seed in range(3):
        pts, boxes = _constructed_points_and_boxes(seed)
        flags = torch.zeros((boxes.shape[0], pts.shape[0]), dtype=torch.int32)
        reg = torch.zeros((pts.shape[0], 3), dtype=torch.float32)
        ext.pts_in_boxes3d(torch.from_numpy(pts), torch.from_numpy(boxes), flags, reg)
        of, orr = OT.pts_in_boxes3d(pts, boxes)
        assert np.array_equal(flags.numpy(), of)
        assert np.array_equal(reg.numpy().view(np.int32), orr.view(np.int32))
        assert (of.sum(0) == 2).any() and of.any(1).all()


def test_oracle_create_target_rules():
    """Forced ties, a GT overlapping no anchor, anchors between the thresholds, the write order."""
    anchors = np.array([[0, 0, -1, 1.6, 3.9, 1.56, 0], [0.2, 0, -1, 1.6, 3.9, 1.56, 0],     # tie for GT 0
                        [5, 0, -1, 1.6, 3.9, 1.56, 0],                                      # between thresholds
                        [40, 0, -1, 1.6, 3.9, 1.56, 0]], f32)                               # background
    gt = np.array([[0.1, 0, -1, 1.6, 3.9, 1.56, 0], [5.6, 0, -1, 1.6, 3.9, 1.56, 0],
                   [-30, 0, -1, 1.6, 3.9, 1.56, 0]], f32)                                   # GT 2 overlaps nothing
    iou = OT.near_iou(anchors, gt)
    assert iou[0, 0] == iou[1, 0] and iou[:, 2].max() == 0
    lab, tgt, m = OT.create_target(anchors, None, gt, np.array([1, 2, 3]), OT.near_iou, 0.99, 0.45)
    assert lab.tolist() == [1, 1, 2, 0]          # anchors 0 / 1 forced by GT 0, anchor 2 forced by GT 1
    assert np.all(tgt[3] == 0) and np.all(tgt[:3, 3:6] == 0)
    lab, _, _ = OT.create_target(anchors, np.array([1, 1, 0, 1], bool), gt[:0], None, OT.near_iou, 0.6, 0.45)
    assert lab.tolist() == [0, 0, -1, 0]         # no GT: every masked anchor is background


def test_train_mode_still_raises_and_configs_carry_train_cfg():
    import sassd_b200 as S
    from sassd_b200.builder import build_detector
    for name in ("car_cfg.py", "multi_cfg.py"):
        cfg = S.Config.fromfile(os.path.join(ROOT, "configs", name))
        assert cfg.train_cfg.rpn.anchor_thr == 0.1 and cfg.train_cfg.extra.assigner.pos_iou_thr == 0.7
        model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
        model.train()
        with pytest.raises(NotImplementedError, match="eval"):
            model(None, [{}], return_loss=True)


# ------------------------------------------------------------------------------------------------------------ GPU
def _model(cfg_name="car_cfg.py"):
    import sassd_b200 as S
    from sassd_b200 import checkpoint
    cfg = S.Config.fromfile(os.path.join(ROOT, "configs", cfg_name))
    model, _, _ = S.build_from_config(cfg, device="cuda:0")
    nc = len(model.class_names)
    sd = checkpoint.make_synthetic_state_dict(0, nc)
    sd.update(_aux_weights())
    checkpoint.load_state_dict_into(model, sd)
    return model


def _frames(B, nc=1, empty=()):
    """Synthetic clouds and their cars as GT (x, y, z_bottom, w, l, h, ry), the draws of synth_cloud."""
    from sassd_b200.synth import CAR_SIZE, GROUND_Z, synth_cloud
    pts, gts, labels = [], [], []
    for b in range(B):
        pts.append(synth_cloud(b))
        rng = np.random.default_rng(b)
        cx, cy, swap = rng.uniform(5.0, 60.0, 12), rng.uniform(-20.0, 20.0, 12), rng.random(12) < 0.5
        w, l, h = CAR_SIZE
        g = np.stack([cx, cy, np.full(12, GROUND_Z), np.full(12, w), np.full(12, l), np.full(12, h),
                      np.where(swap, np.pi / 2, 0.0)], 1).astype(f32)
        if b in empty:
            g = g[:0]
        gts.append(g)
        labels.append((np.arange(len(g)) % nc + 1).astype(np.int64))
    return pts, gts, labels


def _host(t):
    return t.detach().cpu().numpy()


@pytest.mark.gpu
def test_points_in_boxes_bit_identical_to_reference_and_oracle():
    from sassd_b200 import ops
    from sassd_b200.single_stage_heads import stage_gt
    ext = _ref_ext()
    pts0, boxes0 = _constructed_points_and_boxes(0)
    pts1, boxes1 = _constructed_points_and_boxes(1)
    pm = np.concatenate([np.c_[np.zeros(len(pts0)), pts0], np.c_[np.ones(len(pts1)), pts1],
                         np.c_[np.full(50, 2.0), pts1[:50]]]).astype(f32)    # frame 2 has no GT
    gtl = [boxes0, boxes1[::-1].copy(), boxes1[:0]]
    gt, _, _, d_ngt = stage_gt(gtl, None, None, "cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_rows = torch.tensor([len(pm)], dtype=torch.int32, device="cuda")
    lab, off, npos = ops.points_in_boxes(torch.from_numpy(pm).cuda(), d_rows, gt, d_ngt, status)
    lab, off = _host(lab), _host(off)
    ol, oo = OT.aux_targets(pm, gtl)
    assert np.array_equal(lab, ol) and np.array_equal(off.view(np.int32), oo.view(np.int32))
    assert int(npos.item()) == int(ol.sum()) and int(status.item()) == 0 and not lab[-50:].any()
    if ext is not None:
        r0 = 0
        for b, g in enumerate(gtl[:2]):
            p = pm[pm[:, 0] == b, 1:4].copy()
            flags = torch.zeros((len(g), len(p)), dtype=torch.int32)
            reg = torch.zeros((len(p), 3), dtype=torch.float32)
            ext.pts_in_boxes3d(torch.from_numpy(p), torch.from_numpy(g), flags, reg)
            assert np.array_equal(lab[r0:r0 + len(p)], flags.numpy().max(0))
            assert np.array_equal(off[r0:r0 + len(p)].view(np.int32), reg.numpy().view(np.int32))
            r0 += len(p)


def _ref_iou3d():
    """RotateIou3dSimilarity with the BEV overlaps of the reference kernel (oracle/_ref/libiou3d_ref.so's
    boxesoverlapLauncher, built unmodified by build()), or None when it was not built."""
    import ctypes
    path = os.path.join(ROOT, "oracle", "_ref", "libiou3d_ref.so")
    if not os.path.isfile(path):
        return None
    fn = getattr(ctypes.CDLL(path), "_Z20boxesoverlapLauncheriPKfiS0_Pf")
    fn.restype = None
    fn.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]

    def iou(a, g):
        qa = torch.from_numpy(OT.bev_boxes(a)).cuda()
        qg = torch.from_numpy(OT.bev_boxes(g)).cuda()
        out = torch.zeros((qa.shape[0], qg.shape[0]), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        fn(qa.shape[0], qa.data_ptr(), qg.shape[0], qg.data_ptr(), out.data_ptr())   # legacy default stream
        torch.cuda.synchronize()
        return OT.iou3d(a, g, bev=_host(out))
    return iou


def _ulp_diff(a, b):
    a, b = np.asarray(a, f32).view(np.int32).astype(np.int64), np.asarray(b, f32).view(np.int32).astype(np.int64)
    return np.abs(a - b)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name", ["car_cfg.py", "multi_cfg.py"])
def test_loss_points_targets_and_losses_match_the_oracle(cfg_name):
    """On the GPU's own head outputs and guided boxes: labels and max IoUs bit-identical, targets within 2 ulp, losses
    within rel 1e-5; forward(return_loss=True) equals loss_points; two calls give the same bits; detections are
    unchanged by the loss call."""
    model = _model(cfg_name)
    nc = len(model.class_names)
    pts, gts, labels = _frames(3, nc, empty=(1,))
    det0 = model.forward_points(pts)
    res, aux = model.loss_points(pts, gts, labels, return_aux=True)
    res2 = model.loss_points(pts, gts, labels)
    assert all(np.float32(res[k]).tobytes() == np.float32(res2[k]).tobytes() for k in res)
    det1 = model.forward_points(pts)
    for a, b in zip(det0, det1):
        for k in a:
            assert (a[k] is None and b[k] is None) or np.array_equal(a[k], b[k])
    B = len(pts)
    # aux
    fr = _host(aux["frame_rows"])
    n0 = int(fr[-1])
    pm = _host(aux["points_mean"])[:n0]
    ol, oo = OT.aux_targets(pm, gts)
    assert np.array_equal(_host(aux["point_labels"])[:n0], ol)
    assert np.array_equal(_host(aux["point_offsets"])[:n0].view(np.int32), oo.view(np.int32))
    exp = OT.aux_losses(_host(aux["point_cls"])[:n0], _host(aux["point_reg"])[:n0], ol, oo, B)
    # rpn
    anchors = model.anchor_set.anchors
    A = np.broadcast_to(anchors, (B,) + anchors.shape)
    mask = _host(aux["mask"]).astype(bool)
    pos, neg = model.rpn_head.thresholds(model.train_cfg.rpn, model.class_names)
    gcls = [l - 1 for l in labels]
    L, T, M = OT.rpn_targets(A, mask, gts, gcls, labels, pos, neg, nc)
    gl, gt_, gm = _host(aux["rpn_labels"]), _host(aux["rpn_targets"]), _host(aux["rpn_ious"])
    assert np.array_equal(gl, L) and np.array_equal(gm.view(np.int32), M.view(np.int32))
    assert (gl > 0).any() and (gl == -1).any() and ((M > neg[0]) & (M < pos[0])).any()
    assert _ulp_diff(gt_, T).max() <= 2
    head = aux["head"]
    box, cls, dirp = [t.reshape(B, -1, w) for t, w in zip(model.rpn_head._split(head), (7, nc, 2))]
    exp.update(OT.rpn_losses(_host(box), _host(cls), _host(dirp), L, T, A))
    # pswarp: the GPU's guided boxes and scores, GT rows first
    gt_cap = aux["ps_boxes"].shape[1] - aux["guided"].shape[1]
    ref_iou3d = _ref_iou3d()
    boxes, scores = _host(aux["ps_boxes"]), _host(aux["ps_scores"])
    d_k = _host(aux["d_k"])
    olab, oscore = [], []
    for b in range(B):
        sel = np.r_[np.arange(len(gts[b])), gt_cap + np.arange(d_k[b])]
        lb, _, mb = OT.create_target(boxes[b, sel], None, gts[b], None, OT.iou3d, 0.7, 0.7, encode=False)
        glab = _host(aux["ps_labels"])[b]
        assert np.array_equal(glab[sel], lb) and (glab[np.setdiff1d(np.arange(glab.size), sel)] == -1).all()
        assert np.abs(_host(aux["ps_ious"])[b, sel] - mb).max() <= 1e-6
        if ref_iou3d is not None and len(gts[b]):       # the rotated overlaps of the reference kernel, bit for bit
            rl, _, rm = OT.create_target(boxes[b, sel], None, gts[b], None, ref_iou3d, 0.7, 0.7, encode=False)
            assert np.array_equal(glab[sel], rl)
            assert np.array_equal(_host(aux["ps_ious"])[b, sel].view(np.int32), rm.view(np.int32))
        olab.append(lb); oscore.append(scores[b, sel])
    exp.update(OT.pswarp_loss(np.concatenate(oscore), np.concatenate(olab), B))
    for k, v in exp.items():
        assert abs(res[k] - v) <= 1e-5 * max(abs(v), 1e-6), (k, res[k], v)
    assert res["loss_cls"] > 0 and res["aux_loss_reg"] > 0 and res["rpn_loc_loss"] > 0
    # the reference signature on the same voxels
    fr = _host(aux["frame_rows"])
    vox = [aux["voxels"][fr[b]:fr[b + 1]] for b in range(B)]
    coords = [aux["coors"][fr[b]:fr[b + 1], 1:] for b in range(B)]
    nump = [aux["num_points"][fr[b]:fr[b + 1]] for b in range(B)]
    per = anchors.shape[0] // nc
    names = model.class_names
    anc = {n: [torch.from_numpy(anchors[c * per:(c + 1) * per]) for _ in range(B)] for c, n in enumerate(names)}
    msk = {n: [torch.from_numpy(mask[b, c * per:(c + 1) * per]) for b in range(B)] for c, n in enumerate(names)}
    types = [np.array([names[l - 1] for l in lb]) for lb in labels]
    with torch.no_grad():
        ref = model(None, [{}] * B, return_loss=True, voxels=vox, coordinates=coords, num_points=nump, anchors=anc,
                    anchors_mask=msk, gt_bboxes=[torch.from_numpy(g) for g in gts],
                    gt_labels=[torch.from_numpy(l) for l in labels], gt_types=types)
    assert set(ref) == set(res) and all(tuple(v.shape) == (1,) for v in ref.values())
    # the reference signature feeds the dense convs fp32 maps where the fused step keeps split fp16 planes: the head
    # outputs agree to ~1e-6 of scale, not bit for bit
    for k in res:
        assert abs(float(ref[k]) - res[k]) <= 1e-4 * max(abs(res[k]), 1e-6), (k, float(ref[k]), res[k])


@pytest.mark.gpu
def test_gt_capacity_overflow_raises():
    from sassd_b200 import ops
    model = _model()
    pts, gts, labels = _frames(1)
    n = ops._lib.GT_CAP_MAX
    many = np.repeat(gts[0], (n + 1) // len(gts[0]) + 1, 0)[:n + 1]
    with pytest.raises(ops._lib.SassdError, match="GT_CAP"):
        model.loss_points(pts, [many], [np.ones(n + 1, np.int64)])
    ok, aux = model.loss_points(pts, [many[:n]], [np.ones(n, np.int64)], return_aux=True)     # exactly the capacity
    assert all(np.isfinite(v) for v in ok.values())
    # the full GT table against the oracle: labels and IoUs bit for bit, targets within 2 ulp, losses within 2e-6
    anchors = model.anchor_set.anchors
    A = anchors[None]
    mask = _host(aux["mask"]).astype(bool)
    pos, neg = model.rpn_head.thresholds(model.train_cfg.rpn, model.class_names)
    gt1, lab1 = [many[:n]], [np.ones(n, np.int64)]
    L, T, M = OT.rpn_targets(A, mask, gt1, [l - 1 for l in lab1], lab1, pos, neg, 1)
    assert np.array_equal(_host(aux["rpn_labels"]), L)
    assert np.array_equal(_host(aux["rpn_ious"]).view(np.int32), M.view(np.int32))
    assert _ulp_diff(_host(aux["rpn_targets"]), T).max() <= 2
    box, cls, dirp = [t.reshape(1, -1, w) for t, w in zip(model.rpn_head._split(aux["head"]), (7, 1, 2))]
    exp = OT.rpn_losses(_host(box), _host(cls), _host(dirp), L, T, A)
    for k, v in exp.items():
        assert abs(ok[k] - v) <= 2e-6 * abs(v), (k, ok[k], v)
    res = model.loss_points(pts, [g[:0] for g in gts], [l[:0] for l in labels])
    assert res["rpn_loc_loss"] == 0 and res["aux_loss_reg"] == 0 and res["rpn_cls_loss"] > 0


# ------------------------------------------------------------------------------------------------------------ golden
CASES = ("car", "multi")


def _golden(golden_dir, tag):
    z = np.load(os.path.join(golden_dir, "loss.npz"))
    p = tag + "_"
    g = {k[len(p):]: z[k] for k in z.files if k.startswith(p)}
    B = g["box_preds"].shape[0]
    g["gts"] = [g["gt%d" % b] for b in range(B)]
    g["gt_labels"] = [g["gt_labels%d" % b] for b in range(B)]
    g["gt_types"] = [g["gt_types%d" % b] for b in range(B)]
    g["classes"] = [str(c) for c in g["classes"]]
    c = np.r_[0, np.cumsum(g["ps_counts"])]
    g["guided_list"] = [g["guided"][c[b]:c[b + 1]] for b in range(B)]
    g["B"] = B
    return g


def _thr(classes):
    from sassd_b200.config import ConfigDict
    THR = {"Car": (0.6, 0.45), "Pedestrian": (0.5, 0.35), "Cyclist": (0.5, 0.35)}
    rpn = {c: dict(pos_iou_thr=THR[c][0], neg_iou_thr=THR[c][1]) for c in classes}
    rpn.update(similarity_fn="NearestIouSimilarity")
    extra = dict(assigner=dict(pos_iou_thr=0.7, neg_iou_thr=0.7, similarity_fn="RotateIou3dSimilarity"))
    return [THR[c][0] for c in classes], [THR[c][1] for c in classes], ConfigDict(dict(rpn=dict(assigner=rpn),
                                                                                        extra=extra))


def _oracle_golden(g):
    B, classes = g["B"], g["classes"]
    nc = len(classes)
    pos, neg, _ = _thr(classes)
    gcls = [np.array([classes.index(str(t)) for t in ts]) for ts in g["gt_types"]]
    L, T, M = OT.rpn_targets(g["anchors"], g["mask"], g["gts"], gcls, g["gt_labels"], pos, neg, nc)
    pl, po = OT.aux_targets(g["points_mean"], g["gts"])
    ps = [OT.create_target(g["guided_list"][b], None, g["gts"][b], None, OT.iou3d, 0.7, 0.7, encode=False)
          for b in range(B)]
    losses = OT.rpn_losses(g["box_preds"].reshape(B, -1, 7), g["cls_preds"].reshape(B, -1, nc),
                           g["dir_preds"].reshape(B, -1, 2), L, T, g["anchors"])
    losses.update(OT.aux_losses(g["point_cls"], g["point_reg"], pl, po, B))
    losses.update(OT.pswarp_loss(g["ps_scores"], np.concatenate([x[0] for x in ps]), B))
    return L, T, M, pl, po, ps, losses


@pytest.mark.parametrize("tag", CASES)
def test_oracle_reproduces_the_reference_golden(golden_dir, tag):
    g = _golden(golden_dir, tag)
    L, T, M, pl, po, ps, losses = _oracle_golden(g)
    assert np.array_equal(L, g["rpn_labels"]) and np.array_equal(M, g["rpn_ious"])
    assert np.abs(T - g["rpn_targets"]).max() <= 1e-6
    assert np.array_equal(pl, g["point_labels"]) and np.array_equal(po, g["point_offsets"])
    assert np.array_equal(np.concatenate([x[0] for x in ps]), g["ps_labels"])
    assert np.abs(np.concatenate([x[2] for x in ps]) - g["ps_ious"]).max() <= 1e-6
    for k, v in losses.items():
        ref = float(g["loss_" + k][0])
        assert abs(v - ref) <= 1e-6 * abs(ref), (k, v, ref)
    # the cases the fixture was built to hit
    assert (g["rpn_labels"] > 0).any() and (g["rpn_labels"] == 0).any() and (g["rpn_labels"] == -1).any()
    assert (g["point_labels"] == 1).any() and (g["ps_labels"] > 0).any() and (g["ps_labels"] == 0).any()
    assert g["min_gap_to_thr"] < 0.01


@pytest.mark.gpu
@pytest.mark.parametrize("tag", CASES)
def test_kernels_reproduce_the_reference_golden(golden_dir, tag):
    from sassd_b200 import ops
    from sassd_b200.single_stage_heads import PSWarpHead, SSDRotateHead, stage_gt
    g = _golden(golden_dir, tag)
    B, classes = g["B"], g["classes"]
    nc = len(classes)
    pos, neg, cfg = _thr(classes)
    dev = torch.device("cuda")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    status = torch.zeros((1,), dtype=torch.int32, device=dev)
    # points in boxes and the aux loss
    gt, gcls, glab, d_ngt = stage_gt(g["gts"], [np.array([classes.index(str(x)) for x in ts]) for ts in g["gt_types"]],
                                     g["gt_labels"], dev)
    n = len(g["points_mean"])
    d_rows = torch.tensor([n], dtype=torch.int32, device=dev)
    lab, off, npos = ops.points_in_boxes(t(g["points_mean"]), d_rows, gt, d_ngt, status)
    assert np.array_equal(_host(lab), g["point_labels"].astype(np.int32))
    assert np.array_equal(_host(off).view(np.int32), g["point_offsets"].view(np.int32))
    out = torch.zeros((6,), dtype=torch.float32, device=dev)
    ops.aux_loss(t(g["point_cls"].reshape(-1)), t(g["point_reg"]), lab, off, d_rows, B, npos, out[0:2])
    # RPN targets on the reference's per-frame anchors, and the losses through the public signature
    rl, rt, ri, _ = ops.assign_rpn(t(g["anchors"]), t(g["mask"].astype(np.uint8)), nc, gt, gcls, glab, d_ngt, pos, neg,
                                   status)
    assert np.array_equal(_host(rl), g["rpn_labels"].astype(np.int32))
    assert np.array_equal(_host(ri).view(np.int32), g["rpn_ious"].view(np.int32))
    assert _ulp_diff(_host(rt), g["rpn_targets"]).max() <= 2
    head = SSDRotateHead(num_class=nc, num_output_filters=8).to(dev)
    per = g["anchors"].shape[1] // nc
    anc = {c: t(g["anchors"][:, i * per:(i + 1) * per]) for i, c in enumerate(classes)}
    msk = {c: t(g["mask"][:, i * per:(i + 1) * per]) for i, c in enumerate(classes)}
    rpn = head.loss(t(g["box_preds"]), t(g["cls_preds"]), t(g["dir_preds"]), [t(x) for x in g["gts"]],
                    [t(x) for x in g["gt_labels"]], g["gt_types"], anc, msk, cfg.rpn)
    # PSWarp targets on the reference's guided boxes (GT rows first), and its loss
    ks = g["ps_counts"]
    k_cap = int(ks.max())
    boxes = np.zeros((B, k_cap, 7), np.float32)
    for b in range(B):
        boxes[b, :ks[b]] = g["guided_list"][b]
    pl, _, _ = ops.assign_pswarp(gt, d_ngt, t(boxes), t(ks.astype(np.int32)), 0.7, 0.7, status)
    pl = _host(pl)
    assert np.array_equal(np.concatenate([pl[b, :ks[b]] for b in range(B)]), g["ps_labels"].astype(np.int32))
    ps = PSWarpHead((0., 40.), .4, 8, 1, 28).to(dev)
    psl = ps.loss(t(g["ps_scores"]), [t(x) for x in g["gts"]], None, [t(x) for x in g["guided_list"]], cfg.extra)
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    got = dict(aux_loss_cls=float(out[0]), aux_loss_reg=float(out[1]), loss_cls=float(psl["loss_cls"]))
    got.update({k: float(v) for k, v in rpn.items()})
    for k, v in got.items():
        ref = float(g["loss_" + k][0])
        assert abs(v - ref) <= 1e-5 * abs(ref), (k, v, ref)
    ref_iou3d = _ref_iou3d()
    if ref_iou3d is not None:
        for b in range(B):
            _, _, rm = OT.create_target(g["guided_list"][b], None, g["gts"][b], None, ref_iou3d, 0.7, 0.7, encode=False)
            _, gi, _ = ops.assign_pswarp(gt, d_ngt, t(boxes), t(ks.astype(np.int32)), 0.7, 0.7, status)
            assert np.array_equal(_host(gi)[b, :ks[b]].view(np.int32), rm.view(np.int32))

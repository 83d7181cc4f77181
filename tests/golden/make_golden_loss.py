"""Generate tests/golden/loss.npz by running the REFERENCE's own training-target and loss code on the CPU:
create_target_torch, SSDRotateHead.loss, PSWarpHead.loss, SpMiddleFHD.build_aux_target and SpMiddleFHD.aux_loss.
Run once where the original project is checked out and __graft_entry__.build() made oracle/_ref/; the fixture is
committed because neither exists everywhere the tests run.

    python tests/golden/make_golden_loss.py

Under make_golden.py's import stubs, with three substitutions for the reference's native code:
  * Tensor.cuda is the identity and torch.cuda.FloatTensor a CPU zeros tensor (the reference moves targets to the GPU);
  * iou3d_cuda.boxes_overlap_bev_gpu fills its output with oracle_box_overlap (oracle/nms.c, a transcription of the
    reference's box_overlap);
  * points_op_cpu.pts_in_boxes3d is the reference's points_op.cpp, built unmodified by oracle/points_op_ref.py.

Cases, per anchor config (car_cfg: Car; multi_cfg: Car, Pedestrian, Cyclist), two frames on a 16 x 20 cell crop of the
configs' anchor grid: GT boxes that force tied anchors, a GT that overlaps no anchor, GT between the thresholds, a class
without GT in a frame (multi_cfg), random masks and head outputs; points on box faces and corners and inside two boxes;
guided boxes that jitter the GT around the 0.7 threshold.  min |IoU - thr| is recorded per case.
"""
import ctypes
import os
import sys
import types
import unittest.mock  # noqa: F401  (make_golden's stubs)

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

H, W, B = 16, 20, 2
THR = {"Car": (0.6, 0.45), "Pedestrian": (0.5, 0.35), "Cyclist": (0.5, 0.35)}
SIZES = {"Car": [1.6, 3.9, 1.56], "Pedestrian": [0.6, 0.8, 1.73], "Cyclist": [0.6, 1.76, 1.73]}


def install_stubs():
    from make_golden import import_reference_mmdet
    from oracle import points_op_ref
    from oracle import ref_pipeline as R
    import_reference_mmdet()
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.cuda.FloatTensor = lambda size: torch.zeros(tuple(size), dtype=torch.float32)
    pf = ctypes.POINTER(ctypes.c_float)

    def boxes_overlap_bev_gpu(a, b, out):
        a, b = np.ascontiguousarray(a.numpy(), np.float32), np.ascontiguousarray(b.numpy(), np.float32)
        for i in range(a.shape[0]):
            for j in range(b.shape[0]):
                out[i, j] = R.lib().oracle_box_overlap(a[i].ctypes.data_as(pf), b[j].ctypes.data_as(pf))
    sys.modules["mmdet.ops.iou3d.iou3d_cuda"].boxes_overlap_bev_gpu = boxes_overlap_bev_gpu
    ext = points_op_ref.load()
    assert ext is not None, "run __graft_entry__.build() first: it builds the reference points_op extension"
    sys.modules["mmdet.ops.points_op.points_op_cpu"].pts_in_boxes3d = ext.pts_in_boxes3d


def cfg_dict(classes):
    from sassd_b200.config import ConfigDict
    rpn = {c: dict(pos_iou_thr=THR[c][0], neg_iou_thr=THR[c][1], min_pos_iou=THR[c][1]) for c in classes}
    rpn.update(ignore_iof_thr=-1, similarity_fn="NearestIouSimilarity")
    return ConfigDict(dict(rpn=dict(assigner=rpn, anchor_thr=0.1),
                           extra=dict(assigner=dict(pos_iou_thr=0.7, neg_iou_thr=0.7, min_pos_iou=0.7,
                                                    ignore_iof_thr=-1, similarity_fn="RotateIou3dSimilarity"))))


def gt_frames(rng, classes):
    """Two frames of GT (x, y, z_bottom, w, l, h, ry) in the anchor crop x 0.2..7.8, y -39.8..-33.8."""
    gts, types_, labels = [], [], []
    for b in range(B):
        rows, tl = [], []
        # frame 0: a box centred between two anchor rows (tied IoUs), frame 1: a rotated one
        rows.append([1.0 + 0.2 * b, -37.6, -1.78, 1.6, 3.9, 1.56, 0.0 if b == 0 else 1.2]); tl.append("Car")
        rows.append([60.0, 20.0, -1.7, 1.6, 3.9, 1.56, 0.3]); tl.append("Car")            # overlaps no anchor
        rows.append([rng.uniform(2, 7), rng.uniform(-39, -35), -1.7, 1.7, 4.1, 1.5, rng.uniform(-3, 3)])
        tl.append("Car")
        if len(classes) > 1 and b == 0:                   # frame 1 has no Cyclist
            rows.append([rng.uniform(2, 7), rng.uniform(-39, -35), -1.6, 0.6, 1.76, 1.73, 0.0]); tl.append("Cyclist")
        if len(classes) > 1:
            rows.append([rng.uniform(2, 7), rng.uniform(-39, -35), -1.6, 0.6, 0.8, 1.73, np.pi / 2])
            tl.append("Pedestrian")
        rows.append([4.0, -36.0, -1.7, 1.6, 3.9, 1.56, np.pi / 4]); tl.append("Car")     # the > pi/4 swap edge
        gts.append(np.asarray(rows, np.float32))
        types_.append(np.array(tl))
        labels.append(np.array([classes.index(t) + 1 if t in classes else 1 for t in tl], np.int64))
    return gts, types_, labels


def points_for(rng, gts):
    """points_mean [N,4] (b, x, y, z): face and corner points of every box, points inside two boxes, random points."""
    out = []
    for b, g in enumerate(gts):
        p = [np.c_[rng.uniform(0, 9, 600), rng.uniform(-40, -33, 600), rng.uniform(-3, 1, 600)]]
        for bx in g:
            c, s = np.cos(bx[6]), np.sin(bx[6])
            for u in (-0.5, 0.0, 0.5):
                for v in (-0.5, 0.0, 0.5):
                    lx, ly = np.float32(u * bx[3]), np.float32(v * bx[4])
                    p.append([[bx[0] + lx * c - ly * s, bx[1] + lx * s + ly * c, bx[2] + bx[5] * t]
                              for t in (0.0, 0.5, 1.0)])
            p.append(bx[None, :3] + rng.normal(0, 0.4, (60, 3)) * bx[3:6])
        # inside the first and the last box of the frame: centre of their overlap
        p.append([[(g[0, 0] + g[-1, 0]) / 2, (g[0, 1] + g[-1, 1]) / 2, -1.0]])
        q = np.concatenate([np.asarray(x, np.float64).reshape(-1, 3) for x in p]).astype(np.float32)
        out.append(np.c_[np.full(len(q), b, np.float32), q])
    return np.ascontiguousarray(np.concatenate(out).astype(np.float32))


def guided_for(rng, gts):
    """Per frame: GT rows first (as get_guided_anchors prepends them), then jittered copies and random boxes."""
    out = []
    for g in gts:
        j = np.repeat(g, 6, 0) + rng.normal(0, 1, (6 * len(g), 7)).astype(np.float32) * [.15, .15, .05, .05, .1, .05, .1]
        r = np.c_[rng.uniform(0, 9, (20, 1)), rng.uniform(-40, -33, (20, 1)), np.full((20, 1), -1.7),
                  rng.uniform(0.5, 2, (20, 1)), rng.uniform(0.8, 4.5, (20, 1)), rng.uniform(1.4, 1.8, (20, 1)),
                  rng.uniform(-3, 3, (20, 1))]
        out.append(np.concatenate([g, j, r]).astype(np.float32))
    return out


def run_case(tag, classes, seed, out):
    from mmdet.core.anchor.anchor3d_generator import AnchorGeneratorStride
    from mmdet.core.bbox3d.target_ops import create_target_torch
    from mmdet.models.necks.cmn import SpMiddleFHD
    from mmdet.models.single_stage_heads import ssd_rotate_head as RH
    from mmdet.ops.iou3d import iou3d_utils
    rng = np.random.default_rng(seed)
    g = torch.Generator().manual_seed(seed)
    nc = len(classes)
    cfg = cfg_dict(classes)
    anchors, masks = {}, {}
    for c in classes:
        gen = AnchorGeneratorStride(sizes=SIZES[c], anchor_strides=[0.4, 0.4, 1.0], anchor_offsets=[0.2, -39.8, -1.78],
                                    rotations=[0, 1.57])
        a = torch.from_numpy(np.ascontiguousarray(gen([1, H, W]).reshape(-1, 7), np.float32))
        anchors[c] = a[None].repeat(B, 1, 1)
        masks[c] = torch.from_numpy(rng.random((B, a.shape[0])) < 0.85)
    gts, gtypes, glabels = gt_frames(rng, classes)
    gt_t = [torch.from_numpy(x) for x in gts]
    lb_t = [torch.from_numpy(x) for x in glabels]
    head = RH.SSDRotateHead(num_class=nc, num_output_filters=8, num_anchor_per_loc=2, use_sigmoid_cls=True,
                            encode_rad_error_by_sin=True, use_direction_classifier=True, box_code_size=7)
    box = torch.randn((B, nc, H, W, 14), generator=g) * 0.3
    cls = torch.randn((B, nc, H, W, 2 * nc), generator=g) - 2.0
    dirp = torch.randn((B, nc, H, W, 4), generator=g)
    rpn = head.loss(box, cls, dirp, gt_t, lb_t, list(gtypes), anchors, masks, cfg.rpn)
    # the targets the loss used, frame by frame and class by class
    L, T, M, gap = [], [], [], np.inf
    for c in classes:
        gt_mask = [torch.BoolTensor(t == c) for t in gtypes]
        lab, tgt, iou = [], [], []
        for b in range(B):
            l_, t_, m_ = create_target_torch(anchors[c][b], masks[c][b], gt_t[b], lb_t[b], gt_mask[b],
                                             similarity_fn=iou3d_utils.NearestIouSimilarity(),
                                             box_encoding_fn=RH.second_box_encode,
                                             matched_threshold=THR[c][0], unmatched_threshold=THR[c][1], box_code_size=7)
            lab.append(l_.numpy()); tgt.append(t_.numpy())
            mm = np.zeros(anchors[c].shape[1], np.float32)
            if len(m_) == int(masks[c][b].sum()):
                mm[masks[c][b].numpy()] = m_.numpy()
            iou.append(mm)
            if len(m_):
                gap = min(gap, float(np.abs(m_.numpy()[:, None] - np.array(THR[c])[None]).min()))
        L.append(np.stack(lab)); T.append(np.stack(tgt)); M.append(np.stack(iou))
    # aux
    pm = points_for(rng, gts)
    point_cls = torch.randn((len(pm), 1), generator=g)
    point_reg = torch.randn((len(pm), 3), generator=g) * 0.5
    neck = types.SimpleNamespace()
    neck.build_aux_target = lambda nxyz, boxes, enlarge=1.0: SpMiddleFHD.build_aux_target(neck, nxyz, boxes, enlarge)
    p_lab, p_off = neck.build_aux_target(torch.from_numpy(pm), [x.clone() for x in gt_t])
    aux = SpMiddleFHD.aux_loss(neck, torch.from_numpy(pm), point_cls, point_reg, [x.clone() for x in gt_t])
    # pswarp
    guided = guided_for(rng, gts)
    ps = RH.PSWarpHead(grid_offsets=(0., 40.), featmap_stride=.4, in_channels=8, num_class=1, num_parts=28)
    scores = torch.randn((sum(len(x) for x in guided),), generator=g)
    ps_loss = ps.loss(scores, gt_t, lb_t, [torch.from_numpy(x) for x in guided], cfg.extra)
    ps_lab, ps_iou = [], []
    for b in range(B):
        l_, _, m_ = create_target_torch(torch.from_numpy(guided[b]), None, gt_t[b], None, None,
                                        similarity_fn=iou3d_utils.RotateIou3dSimilarity(),
                                        box_encoding_fn=RH.second_box_encode, matched_threshold=0.7,
                                        unmatched_threshold=0.7)
        ps_lab.append(l_.numpy()); ps_iou.append(m_.numpy())
        gap = min(gap, float(np.abs(m_.numpy() - 0.7).min()))
    p = tag + "_"
    out.update({p + "classes": np.array(classes), p + "anchors": np.concatenate([anchors[c].numpy() for c in classes], 1),
                p + "mask": np.concatenate([masks[c].numpy() for c in classes], 1),
                p + "box_preds": box.numpy(), p + "cls_preds": cls.numpy(), p + "dir_preds": dirp.numpy(),
                p + "rpn_labels": np.concatenate(L, 1), p + "rpn_targets": np.concatenate(T, 1),
                p + "rpn_ious": np.concatenate(M, 1),
                p + "points_mean": pm, p + "point_cls": point_cls.numpy(), p + "point_reg": point_reg.numpy(),
                p + "point_labels": p_lab.numpy(), p + "point_offsets": p_off.numpy(),
                p + "ps_scores": scores.numpy(), p + "ps_labels": np.concatenate(ps_lab),
                p + "ps_ious": np.concatenate(ps_iou), p + "ps_counts": np.array([len(x) for x in guided], np.int32),
                p + "guided": np.concatenate(guided), p + "min_gap_to_thr": np.float64(gap)})
    for b in range(B):
        out[p + "gt%d" % b] = gts[b]
        out[p + "gt_labels%d" % b] = glabels[b]
        out[p + "gt_types%d" % b] = gtypes[b]
    for k, v in list(rpn.items()) + list(aux.items()) + list(ps_loss.items()):
        out[p + "loss_" + k] = v.detach().numpy().astype(np.float32)
    print(tag, {k: float(v) for k, v in list(rpn.items()) + list(aux.items()) + list(ps_loss.items())},
          "positives:", int((out[p + "rpn_labels"] > 0).sum()), int(out[p + "point_labels"].sum()),
          int((out[p + "ps_labels"] > 0).sum()), "min |iou - thr|: %.3g" % gap)


def main():
    install_stubs()
    out = {}
    run_case("car", ["Car"], 0, out)
    run_case("multi", ["Car", "Pedestrian", "Cyclist"], 1, out)
    np.savez_compressed(os.path.join(HERE, "loss.npz"), **out)


if __name__ == "__main__":
    main()

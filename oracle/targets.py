"""ORACLE: numpy restatement of SA-SSD's training targets and losses (forward only) — test infrastructure only.

* ``pts_in_boxes3d`` / ``aux_targets``: points_op.cpp:92-144 and cmn.py:44-70, with the C++ expression types (double
  half sizes, cz rounded to float, double cos / sin stored to float, fp32 rotation without contraction, the z centre
  from the box's fourth value).
* ``create_target``: target_ops.py:139-277 over a dense IoU matrix, with ``near_iou`` (NearestIouSimilarity) or
  ``iou3d`` (RotateIou3dSimilarity; the BEV overlap is oracle_box_overlap of nms.c, the reference's box_overlap).
* ``rpn_losses`` / ``pswarp_loss`` / ``aux_losses``: ssd_rotate_head.py:160-305,450-485, cmn.py:72-100,
  losses.py:31-114.  Elements are fp32, sums fp64.

A frame without GT is all background (aux labels 0, masked anchors 0).
"""
import ctypes

import numpy as np

from . import ref_pipeline as R

f32 = np.float32
PI_F = f32(np.pi)


# ---------------------------------------------------------------------------------------------------- aux targets
def pts_in_boxes3d(pts, boxes):
    """pts [N,3], boxes [M,7] float32 -> (flags [M,N] int32, reg [N,3] float32)."""
    pts = np.ascontiguousarray(pts, f32).reshape(-1, 3)
    boxes = np.ascontiguousarray(boxes, f32).reshape(-1, 7)
    N = pts.shape[0]
    flags = np.zeros((boxes.shape[0], N), np.int32)
    reg = np.zeros((N, 3), f32)
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    for i, b in enumerate(boxes):
        cx, cy, bz, w, l, h, ang = [f32(v) for v in b]
        cz = f32(np.float64(bz) + np.float64(h) / 2.0)
        hh = np.float64(h) / 2.0
        near = ~((np.abs(x - cx) > f32(10.0)) | (np.abs(z - cz).astype(np.float64) > hh) | (np.abs(y - cy) > f32(10.0)))
        cosa, sina = f32(np.cos(np.float64(ang))), f32(np.sin(np.float64(ang)))
        dx, dy = x - cx, y - cy
        x_rot = (dx * cosa) + (dy * -sina)
        y_rot = (dx * sina) + (dy * cosa)
        xr, yr = x_rot.astype(np.float64), y_rot.astype(np.float64)
        inside = near & (xr >= -np.float64(w) / 2.0) & (xr <= np.float64(w) / 2.0) & \
            (yr >= -np.float64(l) / 2.0) & (yr <= np.float64(l) / 2.0)
        flags[i] = inside
        reg[inside, 0] = x[inside] - cx
        reg[inside, 1] = y[inside] - cy
        reg[inside, 2] = (z[inside].astype(np.float64) - (np.float64(bz) + np.float64(w) / 2.0)).astype(f32)
    return flags, reg


def aux_targets(points_mean, gt_bboxes):
    """points_mean [N,4] (b, x, y, z), frames in row order -> (labels [N] uint8, offsets [N,3])."""
    labels, offsets = [], []
    for b, g in enumerate(gt_bboxes):
        xyz = points_mean[points_mean[:, 0] == b, 1:4]
        flags, reg = pts_in_boxes3d(xyz, g)
        labels.append(flags.max(0).astype(np.uint8) if flags.shape[0] else np.zeros(len(xyz), np.uint8))
        offsets.append(reg)
    return np.concatenate(labels), np.concatenate(offsets)


# ---------------------------------------------------------------------------------------------------- similarities
def near_boxes(boxes):
    b = np.asarray(boxes, f32).reshape(-1, 7)
    rot = b[:, 6]
    lp = rot - np.floor(rot / PI_F + f32(0.5)) * PI_F
    swap = np.abs(lp) > f32(np.pi / 4)
    dx = np.where(swap, b[:, 4], b[:, 3])
    dy = np.where(swap, b[:, 3], b[:, 4])
    return np.stack([b[:, 0] - dx / f32(2), b[:, 1] - dy / f32(2), b[:, 0] + dx / f32(2), b[:, 1] + dy / f32(2)], 1)


def near_iou(anchors, gt):
    """NearestIouSimilarity [Na,G] fp32."""
    a, g = near_boxes(anchors), near_boxes(gt)
    lt = np.maximum(a[:, None, :2], g[None, :, :2])
    rb = np.minimum(a[:, None, 2:], g[None, :, 2:])
    wh = np.maximum(rb - lt, f32(0))
    ov = wh[..., 0] * wh[..., 1]
    a1 = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    a2 = (g[:, 2] - g[:, 0]) * (g[:, 3] - g[:, 1])
    return ov / ((a1[:, None] + a2[None, :]) - ov)


def bev_boxes(boxes):
    b = np.asarray(boxes, f32).reshape(-1, 7)
    return np.ascontiguousarray(np.stack([b[:, 0] - b[:, 3] / f32(2), b[:, 1] - b[:, 4] / f32(2),
                                          b[:, 0] + b[:, 3] / f32(2), b[:, 1] + b[:, 4] / f32(2), b[:, 6]], 1))


def overlap_bev(a, b):
    """box_overlap of every pair, [Na,Nb] (oracle_box_overlap, nms.c)."""
    qa, qb = bev_boxes(a), bev_boxes(b)
    L = R.lib()
    out = np.zeros((qa.shape[0], qb.shape[0]), f32)
    pf = ctypes.POINTER(ctypes.c_float)
    for i in range(qa.shape[0]):
        for j in range(qb.shape[0]):
            out[i, j] = L.oracle_box_overlap(qa[i].ctypes.data_as(pf), qb[j].ctypes.data_as(pf))
    return out


def iou3d(a, b, bev=None):
    """RotateIou3dSimilarity [Na,Nb] fp32; ``bev`` overrides the BEV overlaps (e.g. the reference kernel's)."""
    a, b = np.asarray(a, f32).reshape(-1, 7), np.asarray(b, f32).reshape(-1, 7)
    ov_bev = overlap_bev(a, b) if bev is None else bev
    top = np.minimum((a[:, 2] + a[:, 5])[:, None], (b[:, 2] + b[:, 5])[None, :])
    oh = np.maximum(top - np.maximum(a[:, 2][:, None], b[:, 2][None, :]), f32(0))
    ov = ov_bev * oh
    va = (a[:, 3] * a[:, 4]) * a[:, 5]
    vb = (b[:, 3] * b[:, 4]) * b[:, 5]
    return ov / np.maximum((va[:, None] + vb[None, :]) - ov, f32(1e-7))


def box_encode(g, a):
    """second_box_encode, fp32."""
    g, a = np.asarray(g, f32).reshape(-1, 7), np.asarray(a, f32).reshape(-1, 7)
    zg = g[:, 2] + g[:, 5] / f32(2)
    za = a[:, 2] + a[:, 5] / f32(2)
    diag = np.sqrt(a[:, 4] * a[:, 4] + a[:, 3] * a[:, 3])
    return np.stack([(g[:, 0] - a[:, 0]) / diag, (g[:, 1] - a[:, 1]) / diag, (zg - za) / a[:, 5],
                     np.log(g[:, 3] / a[:, 3]), np.log(g[:, 4] / a[:, 4]), np.log(g[:, 5] / a[:, 5]),
                     g[:, 6] - a[:, 6]], 1).astype(f32)


# ---------------------------------------------------------------------------------------------------- assignment
def create_target(anchors, mask, gt, gt_classes, iou_fn, pos_thr, neg_thr, encode=True):
    """create_target_torch for one frame (and class).  Returns (labels [Na] int64, targets [Na,7], max_iou [Na])."""
    anchors = np.asarray(anchors, f32).reshape(-1, 7)
    Na = anchors.shape[0]
    mask = np.ones(Na, bool) if mask is None else np.asarray(mask, bool)
    inds = np.nonzero(mask)[0]
    a = anchors[inds]
    gt = np.asarray(gt, f32).reshape(-1, 7)
    gt_classes = np.ones(len(gt), np.int64) if gt_classes is None else np.asarray(gt_classes, np.int64)
    n = len(inds)
    labels = np.full(n, -1, np.int64)
    targets = np.zeros((n, 7), f32)
    amax = np.zeros(n, f32)
    if len(gt) and n:
        ov = iou_fn(a, gt)
        arg = ov.argmax(1)
        amax = ov[np.arange(n), arg]
        gmax = ov.max(0)
        gmax = np.where(gmax == 0, f32(-1), gmax)
        forced = (ov == gmax[None, :]).any(1)
        labels[forced] = gt_classes[arg[forced]]
        pos = amax >= pos_thr
        labels[pos] = gt_classes[arg[pos]]
        fg = labels > 0
        labels[amax < neg_thr] = 0
        labels[forced] = gt_classes[arg[forced]]
        if encode and fg.any():
            targets[fg] = box_encode(gt[arg[fg]], a[fg])
    else:
        labels[:] = 0
    L = np.full(Na, -1, np.int64)
    L[inds] = labels
    T = np.zeros((Na, 7), f32)
    T[inds] = targets
    M = np.zeros(Na, f32)
    M[inds] = amax
    return L, T, M


# ---------------------------------------------------------------------------------------------------- losses
def _sig(x):
    return (f32(1) / (f32(1) + np.exp(-x.astype(f32)))).astype(f32)


def focal(x, t, w):
    """sigmoid_focal_loss elements, gamma 2, alpha 0.25, fp32."""
    x, t, w = np.asarray(x, f32), np.asarray(t, f32), np.asarray(w, f32)
    p = _sig(x)
    pt = (f32(1) - p) * t + p * (f32(1) - t)
    wt = (f32(0.25) * t + f32(0.75) * (f32(1) - t)) * w
    wt = wt * (pt * pt)
    bce = np.maximum(x, f32(0)) - x * t + np.log1p(np.exp(-np.abs(x)))
    return (bce * wt).astype(f32)


def smooth_l1(p, t):
    beta = f32(1.0 / 9.0)
    d = np.abs(np.asarray(p, f32) - np.asarray(t, f32))
    return np.where(d < beta, f32(0.5) * d * d / beta, d - f32(0.5 / 9.0)).astype(f32)


def ce2(logits, label):
    lg = np.asarray(logits, f32)
    m = lg.max(-1)
    lse = m + np.log(np.exp(lg[..., 0] - m) + np.exp(lg[..., 1] - m))
    return (lse - np.take_along_axis(lg, label[..., None].astype(np.int64), -1)[..., 0]).astype(f32)


def _sum(x):
    return float(np.sum(np.asarray(x, np.float64)))


def rpn_losses(box_preds, cls_preds, dir_preds, labels, targets, anchors):
    """box_preds [B,Na,7], cls_preds [B,Na,nc], dir_preds [B,Na,2], labels [B,Na], targets [B,Na,7], anchors [B,Na,7]
    -> dict(rpn_loc_loss, rpn_cls_loss, rpn_dir_loss) floats."""
    B = box_preds.shape[0]
    nc = cls_preds.shape[-1]
    pos = (labels > 0).astype(f32)
    cared = (labels >= 0).astype(f32)
    n = np.maximum(pos.sum(1, keepdims=True), f32(1))
    wc, wr = cared / n, pos / n
    onehot = (labels[..., None] == np.arange(1, nc + 1)[None, None, :]).astype(f32)
    cls = _sum(focal(cls_preds, onehot, wc[..., None]))
    bp, tg = np.asarray(box_preds, f32).copy(), np.asarray(targets, f32).copy()
    p6, t6 = bp[..., 6].copy(), tg[..., 6].copy()
    bp[..., 6] = np.sin(p6) * np.cos(t6)
    tg[..., 6] = np.cos(p6) * np.sin(t6)
    loc = _sum(smooth_l1(bp, tg) * wr[..., None])
    dl = ((targets[..., 6] + anchors[..., 6]) > 0).astype(np.int64)
    d = _sum(ce2(dir_preds, dl) * wr)
    return dict(rpn_loc_loss=float(f32(f32(loc) / f32(B)) * f32(2)), rpn_cls_loss=float(f32(cls) / f32(B)),
                rpn_dir_loss=float(f32(f32(d) / f32(B)) * f32(0.2)))


def pswarp_loss(scores, labels, batch):
    labels = np.asarray(labels).reshape(-1)
    w = (labels >= 0).astype(f32) / np.maximum(f32((labels > 0).sum()), f32(1))
    return dict(loss_cls=float(f32(_sum(focal(np.asarray(scores, f32).reshape(-1), (labels > 0).astype(f32), w)))
                               / f32(batch)))


def aux_losses(point_cls, point_reg, labels, offsets, batch):
    labels = np.asarray(labels).reshape(-1)
    pos = (labels > 0).astype(f32)
    n = np.maximum(pos.sum(), f32(1))
    c = _sum(focal(np.asarray(point_cls, f32).reshape(-1), pos, np.ones_like(pos) / n))
    r = _sum(smooth_l1(point_reg, offsets) * (pos / n)[:, None])
    return dict(aux_loss_cls=float(f32(c) / f32(batch)), aux_loss_reg=float(f32(r) / f32(batch)))


def rpn_targets(anchors, masks, gt_bboxes, gt_class, gt_labels, pos_thr, neg_thr, num_class):
    """Per frame and class (anchors [B,Na,7] classes concatenated, masks [B,Na]) -> labels [B,Na], targets, ious."""
    B, Na = masks.shape
    per = Na // num_class
    L = np.full((B, Na), -1, np.int64)
    T = np.zeros((B, Na, 7), f32)
    M = np.zeros((B, Na), f32)
    for b in range(B):
        g = np.asarray(gt_bboxes[b], f32).reshape(-1, 7)
        gc = np.asarray(gt_class[b]).reshape(-1)
        gl = np.asarray(gt_labels[b]).reshape(-1)
        for c in range(num_class):
            sl = slice(c * per, (c + 1) * per)
            sel = gc == c
            L[b, sl], T[b, sl], M[b, sl] = create_target(anchors[b, sl], masks[b, sl], g[sel], gl[sel], near_iou,
                                                         pos_thr[c], neg_thr[c])
    return L, T, M

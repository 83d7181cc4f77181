"""``mmdet.models.single_stage_heads`` mirror for the hot path: SSDRotateHead and
PSWarpHead (mmdet/models/single_stage_heads/ssd_rotate_head.py:95-125,218-235,
307-372,416-447,487-533) plus the NMS wrappers they call
(mmdet/core/post_processing/bbox_nms.py:4-27, mmdet/ops/iou3d/iou3d_utils.py:47-60,114-128).

The losses (``SSDRotateHead.loss``, ``PSWarpHead.loss``) and their target assignment run forward only, on the
device (csrc/targets.cu), for a model in eval() mode.
"""

import numpy as np
import torch
from torch import nn

from . import ops
from .necks import conv2d_nhwc, pack_conv2d_weight
from .spconv import _versions, fold_bn


def _pad_lists(tensors, k_cap, width, dtype, device):
    B = len(tensors)
    out = torch.zeros((B, k_cap) + ((width,) if width else ()), dtype=dtype, device=device)
    for b, t in enumerate(tensors):
        if t is not None and len(t):
            out[b, : len(t)] = t.to(device=device, dtype=dtype)
    return out


def stage_gt(gt_bboxes, gt_class, gt_labels, device):
    """Per-frame ground truth -> the loss kernels' padded layout: gt [B,gt_cap,7] f32, gt_class / gt_label [B,gt_cap]
    i32 and d_ngt [B] i32.  gt_cap is the batch's largest count, at most the kernels' capacity SASSD_GT_CAP_MAX; d_ngt
    holds the true counts, so a frame with more boxes sets SASSD_FLAG_GT_CAP on the device and the caller raises.
    ``gt_class`` (anchor class index per box, -1 none) and ``gt_labels`` default to 0 and 1."""
    t = lambda a: torch.from_numpy(a).to(device)       # noqa: E731
    return tuple(t(a) for a in gt_arrays(gt_bboxes, gt_class, gt_labels))


def gt_arrays(gt_bboxes, gt_class, gt_labels, gt_cap=None):
    """stage_gt's layout on the host: numpy (gt, gt_class, gt_label, n).  ``gt_cap`` defaults to the batch's largest
    count; a captured step passes its fixed SASSD_GT_CAP_MAX."""
    B = len(gt_bboxes)
    gt_bboxes = [(g.detach().cpu().numpy() if torch.is_tensor(g) else np.asarray(g)).reshape(-1, 7) for g in gt_bboxes]
    if gt_cap is None:
        gt_cap = min(max([1] + [g.shape[0] for g in gt_bboxes]), ops._lib.GT_CAP_MAX)
    gt = np.zeros((B, gt_cap, 7), np.float32)
    cls = np.zeros((B, gt_cap), np.int32)
    lab = np.ones((B, gt_cap), np.int32)
    n = np.zeros((B,), np.int32)
    for b, g in enumerate(gt_bboxes):
        n[b] = g.shape[0]
        k = min(g.shape[0], gt_cap)
        gt[b, :k] = g[:k]
        if gt_class is not None:
            cls[b, :k] = np.asarray(gt_class[b]).reshape(-1)[:k]
        if gt_labels is not None:
            lv = gt_labels[b]
            lab[b, :k] = (lv.detach().cpu().numpy() if torch.is_tensor(lv) else np.asarray(lv)).reshape(-1)[:k]
    return gt, cls, lab, n


def _as_class_dict(v):
    return v if isinstance(v, dict) else {None: v}


class SSDRotateHead(nn.Module):
    """Constructor kwargs as in configs/car_cfg.py:16-25."""

    def __init__(self, num_class=1, num_output_filters=768, num_anchor_per_loc=2, use_sigmoid_cls=True,
                 encode_rad_error_by_sin=True, use_direction_classifier=True, box_coder="GroundBox3dCoder",
                 box_code_size=7):
        super().__init__()
        if not (use_sigmoid_cls and use_direction_classifier and box_code_size == 7):
            raise NotImplementedError("SA-SSD configs: sigmoid classification, direction classifier, 7-value box code")
        num_anchor_per_loc *= num_class
        self._num_class = num_class
        self._num_anchor_per_loc = num_anchor_per_loc
        self._use_direction_classifier = use_direction_classifier
        self._use_sigmoid_cls = use_sigmoid_cls
        self._encode_rad_error_by_sin = encode_rad_error_by_sin
        self._box_code_size = box_code_size
        self._num_output_filters = num_output_filters
        self.conv_cls = nn.Conv2d(num_output_filters, num_anchor_per_loc * num_class, 1)
        self.conv_box = nn.Conv2d(num_output_filters, num_anchor_per_loc * box_code_size, 1)
        self.conv_dir_cls = nn.Conv2d(num_output_filters, num_anchor_per_loc * 2, 1)
        self.precision = ops.DEFAULT_PRECISION
        self._packed = None
        self.k_cap = 8192   # guided anchors kept per frame (overflow raises SASSD_FLAG_GUIDED_CAP)

    # channel layout of the fused head map: conv_box | conv_cls | conv_dir_cls
    @property
    def head_channels(self):
        na = self._num_anchor_per_loc
        return na * 7 + na * self._num_class + na * 2

    def _weights(self):
        ver = _versions(self.conv_box.weight, self.conv_cls.weight, self.conv_dir_cls.weight, self.conv_box.bias,
                        self.conv_cls.bias, self.conv_dir_cls.bias)
        if self._packed is None or self._packed[0] != ver:
            w = torch.cat([self.conv_box.weight, self.conv_cls.weight, self.conv_dir_cls.weight], 0)
            b = torch.cat([self.conv_box.bias, self.conv_cls.bias, self.conv_dir_cls.bias], 0)
            self._packed = (ver, pack_conv2d_weight(w), b.detach().float().contiguous())
        return self._packed[1], self._packed[2]

    def forward_nhwc(self, x):
        """x [B,H,W,256] -> fused head map [B,H,W,head_channels] (the three 1x1 convs in one GEMM)."""
        w, b = self._weights()
        return conv2d_nhwc(x, w, None, b, False, self.head_channels, self.precision)

    def _split(self, head):
        B, H, W, _ = head.shape
        na, nc = self._num_anchor_per_loc, self._num_class
        o1, o2 = na * 7, na * 7 + na * nc
        # view(N, ncls, -1, H, W).permute(0,1,3,4,2)  ==  NHWC channel block viewed as [ncls, per_class]
        box = head[..., :o1].reshape(B, H, W, nc, -1).permute(0, 3, 1, 2, 4)
        cls = head[..., o1:o2].reshape(B, H, W, nc, -1).permute(0, 3, 1, 2, 4)
        dirp = head[..., o2:o2 + na * 2].reshape(B, H, W, nc, -1).permute(0, 3, 1, 2, 4)
        return box, cls, dirp

    def forward(self, x):
        """x [B,256,H,W] -> (box [B,ncls,H,W,14], cls [B,ncls,H,W,2*ncls], dir [B,ncls,H,W,4])
        (ssd_rotate_head.py:218-235)."""
        ops.require_cuda()
        head = self.forward_nhwc(x.permute(0, 2, 3, 1).contiguous())
        self._last_head = head
        return self._split(head)

    def _as_head_map(self, box_preds, cls_preds, dir_cls_preds):
        head = getattr(self, "_last_head", None)
        if head is not None and box_preds.untyped_storage().data_ptr() == head.untyped_storage().data_ptr():
            return head
        B, nc, H, W, _ = box_preds.shape
        parts = [t.permute(0, 2, 3, 1, 4).reshape(B, H, W, -1) for t in (box_preds, cls_preds, dir_cls_preds)]
        return torch.cat(parts, -1).contiguous().float()

    def guided_anchors_device(self, head, anchors, anchors_mask, thr, status):
        """No-sync path: head map -> (boxes [B,k_cap,7], labels, anchor index, d_k [B])."""
        # [Na,7] = one table for the batch (fused path); [B,Na,7] = per-frame tables (reference signature)
        return ops.decode_select(head, self._num_class, anchors.contiguous().float(),
                                 anchors_mask.to(torch.uint8).contiguous(), float(thr), self.k_cap, status)

    def thresholds(self, cfg, names):
        """(pos, neg) IoU thresholds per anchor class from train_cfg.rpn (``names``: the anchor classes in order; None =
        the single class of the config)."""
        a = cfg.assigner
        if names == [None]:
            keys = [k for k, v in a.items() if isinstance(v, dict)]
            names = keys[:1]
        return [float(a[k]["pos_iou_thr"]) for k in names], [float(a[k]["neg_iou_thr"]) for k in names]

    def assign(self, anchors, mask, gt, gt_class, gt_label, d_ngt, pos_thr, neg_thr, status):
        """No-sync path: the RPN targets (create_target_torch with NearestIouSimilarity, per frame and class).  anchors
        [Na,7] or [B,Na,7], classes concatenated; mask [B,Na] u8.  Returns (labels, targets, ious, d_npos).  They read
        no prediction, so the checkpoints of one config share them (detectors.CheckpointSweep)."""
        return ops.assign_rpn(anchors.contiguous().float(), mask.to(torch.uint8).contiguous(), self._num_class, gt,
                              gt_class, gt_label, d_ngt, pos_thr, neg_thr, status)

    def loss_device(self, head, anchors, mask, gt, gt_class, gt_label, d_ngt, pos_thr, neg_thr, out, status,
                    targets=None):
        """No-sync path: the targets (assign, or ``targets`` when it already ran on these inputs) and the three RPN
        losses into out[0:3].  Returns assign's (labels, targets, ious, d_npos)."""
        res = self.assign(anchors, mask, gt, gt_class, gt_label, d_ngt, pos_thr, neg_thr, status) \
            if targets is None else targets
        ops.rpn_loss(head, self._num_class, anchors.contiguous().float(), res[0], res[1], res[3], out)
        return res

    def loss(self, box_preds, cls_preds, dir_cls_preds, gt_bboxes, gt_labels, gt_types, anchors, anchors_mask, cfg):
        """ssd_rotate_head.py:261-305: dict(rpn_loc_loss, rpn_cls_loss, rpn_dir_loss), each a [1] tensor.  ``anchors``
        / ``anchors_mask``: per-class dicts of [B,Na_c,7] / [B,Na_c] (the training dataset's), or one tensor for a
        single class.  ``gt_types``: per frame the class name of each box; a box counts for the anchors of its class.
        Thresholds from ``cfg`` (train_cfg.rpn).  A frame without boxes of a class has every masked anchor of that
        class as background."""
        ops.require_cuda()
        anchors, anchors_mask = _as_class_dict(anchors), _as_class_dict(anchors_mask)
        names = list(anchors.keys())
        head = self._as_head_map(box_preds, cls_preds, dir_cls_preds)
        dev, B = head.device, head.shape[0]
        a = torch.cat([anchors[k].to(dev).float().reshape(B, -1, 7) for k in names], 1).contiguous()
        m = torch.cat([anchors_mask[k].to(dev).reshape(B, -1).to(torch.uint8) for k in names], 1).contiguous()
        if names == [None] or gt_types is None:
            gt_class = [np.zeros(len(g), np.int32) for g in gt_bboxes]
        else:
            index = {k: i for i, k in enumerate(names)}
            gt_class = [np.array([index.get(str(t), -1) for t in np.asarray(ts).reshape(-1)], np.int32)
                        for ts in gt_types]
        gt, gcls, glab, d_ngt = stage_gt(gt_bboxes, gt_class, gt_labels, dev)
        pos, neg = self.thresholds(cfg, names)
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        out = torch.zeros((3,), dtype=torch.float32, device=dev)
        self.loss_device(head, a, m, gt, gcls, glab, d_ngt, pos, neg, out, status)
        ops._lib.raise_on_status(status)
        return dict(rpn_loc_loss=out[0:1], rpn_cls_loss=out[1:2], rpn_dir_loss=out[2:3])

    def get_guided_anchors(self, box_preds, cls_preds, dir_cls_preds, anchors, anchors_mask, gt_bboxes, gt_labels,
                           thr=.1):
        """Reference signature (ssd_rotate_head.py:307-372).  With ``gt_bboxes`` / ``gt_labels`` (training) each frame's
        boxes and labels are prepended to its selected boxes and labels (:364-367)."""
        if isinstance(anchors, dict):
            anchors = torch.cat([v for v in anchors.values()], 1)
        if isinstance(anchors_mask, dict):
            anchors_mask = torch.cat([v for v in anchors_mask.values()], 1)
        head = self._as_head_map(box_preds, cls_preds, dir_cls_preds)
        status = torch.zeros((1,), dtype=torch.int32, device=head.device)
        boxes, labels, index, d_k = self.guided_anchors_device(head, anchors, anchors_mask.view(head.shape[0], -1),
                                                               thr, status)
        ks = d_k.tolist()
        ops._lib.raise_on_status(status)
        guided, lbls = [boxes[b, :k] for b, k in enumerate(ks)], [labels[b, :k].long() for b, k in enumerate(ks)]
        if gt_bboxes is not None:
            dev = head.device
            guided = [torch.cat([torch.as_tensor(g).to(dev).float().reshape(-1, 7), x], 0)
                      for g, x in zip(gt_bboxes, guided)]
            lbls = [torch.cat([torch.as_tensor(l).to(dev).long().reshape(-1), x], 0) for l, x in zip(gt_labels, lbls)]
        return guided, lbls


def boxes3d_to_bev_torch(boxes3d):
    """iou3d_utils.py:47-60 (pure indexing; kept for API parity — the fused NMS does this in-kernel)."""
    out = boxes3d.new_empty((boxes3d.shape[0], 5))
    cu, cv = boxes3d[:, 0], boxes3d[:, 1]
    hl, hw = boxes3d[:, 3] / 2, boxes3d[:, 4] / 2
    out[:, 0], out[:, 1] = cu - hl, cv - hw
    out[:, 2], out[:, 3] = cu + hl, cv + hw
    out[:, 4] = boxes3d[:, 6]
    return out


def nms_gpu(boxes, scores, thresh):
    """iou3d_utils.py:114-128: boxes [N,5] BEV, scores [N] -> kept indices, best first.
    Sort is stable (ties keep input order); the greedy sweep runs on the device."""
    ops.require_cuda()
    order = torch.sort(scores, descending=True, stable=True)[1]
    b = boxes[order].contiguous().float()
    keep, d_n = ops.nms_sorted(b, float(thresh))
    return order[keep[: int(d_n.item())]].contiguous()


def rotate_nms_torch(rbboxes, scores, pre_max_size=None, post_max_size=None, iou_threshold=0.5):
    """bbox_nms.py:4-27."""
    if pre_max_size is not None:
        pre_max_size = min(scores.shape[0], pre_max_size)
        scores, indices = torch.topk(scores, k=pre_max_size)
        rbboxes = rbboxes[indices]
    if len(rbboxes) == 0:
        keep = torch.empty((0,), dtype=torch.int64)
    else:
        keep = nms_gpu(rbboxes, scores, iou_threshold)[:post_max_size]
    if keep.shape[0] == 0:
        return None
    return indices[keep] if pre_max_size is not None else keep


class PSWarpHead(nn.Module):
    """Constructor kwargs as in configs/car_cfg.py:26-33."""

    def __init__(self, grid_offsets, featmap_stride, in_channels, num_class=1, num_parts=49):
        super().__init__()
        if num_class * num_parts != 28:
            raise NotImplementedError("the reference's sampling window is hard-coded to 4x7 = 28 parts "
                                      "(ssd_rotate_head.py:374)")
        self._num_class = num_class
        out_channels = num_class * num_parts
        self.grid_offsets = (float(grid_offsets[0]), float(grid_offsets[1]))
        self.spatial_scale = 1.0 / featmap_stride
        self.convs = nn.Sequential(
            nn.Conv2d(in_channels, out_channels, 3, 1, padding=1, bias=False),
            nn.BatchNorm2d(out_channels, eps=1e-3, momentum=0.01),
            nn.ReLU(inplace=True),
            nn.Conv2d(out_channels, out_channels, 1, 1, padding=0, bias=False),
        )
        self.precision = ops.DEFAULT_PRECISION
        self._packed = None
        self.det_cap = 512

    def _weights(self):
        ver = _versions(self.convs[0].weight, self.convs[3].weight)
        if self._packed is None or self._packed[0] != ver:
            self._packed = (ver, pack_conv2d_weight(self.convs[0].weight), pack_conv2d_weight(self.convs[3].weight))
        return self._packed[1], self._packed[2]

    def convs_nhwc(self, x):
        """conv 3x3 + BN + ReLU + conv 1x1 (ssd_rotate_head.py:424-429) on NHWC."""
        if self.training:
            raise NotImplementedError("sassd_b200 is inference-only: call .eval()")
        w0, w1 = self._weights()
        scale, shift = fold_bn(self.convs[1])
        c = self.convs[0].out_channels
        y = conv2d_nhwc(x, w0, scale, shift, True, c, self.precision, split_out=isinstance(x, ops.SplitMap))
        return conv2d_nhwc(y, w1, None, None, False, c, self.precision)

    def forward_device(self, conv6_nhwc, boxes, d_k):
        return self.sample(self.convs_nhwc(conv6_nhwc), boxes, d_k)

    def sample(self, feat, boxes, d_k):
        """Scores of boxes [B,k_cap,7] (d_k [B] of them per frame) on the part-score map of convs_nhwc."""
        return ops.pswarp(feat, boxes, d_k, self.grid_offsets[0], self.grid_offsets[1], self.spatial_scale)

    def loss_device(self, scores, boxes, d_k, gt, d_ngt, cfg, out, status, d_head=None, head_cap=0):
        """No-sync path: targets (create_target_torch with RotateIou3dSimilarity) of box slots [B,n,7] (slots below
        ``head_cap`` hold d_head[b] boxes, the rest d_k[b]; ops.assign_pswarp) and the focal loss of their scores
        [B,n] into out[0].  Returns (labels, ious, d_npos)."""
        a = cfg.assigner
        res = ops.assign_pswarp(gt, d_ngt, boxes, d_k, float(a.pos_iou_thr), float(a.neg_iou_thr), status,
                                d_head=d_head, head_cap=head_cap)
        ops.pswarp_loss(scores.contiguous(), res[0], res[2], out)
        return res

    def loss(self, cls_preds, gt_bboxes, gt_labels, anchors, cfg):
        """ssd_rotate_head.py:450-485: dict(loss_cls=[1] tensor).  ``cls_preds``: forward(is_test=False)'s scores of
        the guided boxes ``anchors`` (one [K_b,7] tensor per frame, GT rows first as get_guided_anchors prepends them),
        concatenated; thresholds from ``cfg`` (train_cfg.extra).  The focal loss is normalised by the positives of the
        whole batch."""
        ops.require_cuda()
        dev = cls_preds.device
        B = len(anchors)
        ks = [len(g) for g in anchors]
        k_cap = max(1, max(ks))
        boxes = _pad_lists([g.view(-1, 7) for g in anchors], k_cap, 7, torch.float32, dev)
        scores = _pad_lists(list(torch.split(cls_preds.reshape(-1), ks)), k_cap, 0, torch.float32, dev)
        d_k = torch.tensor(ks, dtype=torch.int32, device=dev)
        gt, _, _, d_ngt = stage_gt(gt_bboxes, None, None, dev)
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        out = torch.zeros((1,), dtype=torch.float32, device=dev)
        self.loss_device(scores, boxes, d_k, gt, d_ngt, cfg, out, status)
        ops._lib.raise_on_status(status)
        return dict(loss_cls=out)

    def forward(self, x, guided_anchors, is_test=False):
        """Reference signature (ssd_rotate_head.py:431-447): x [B,256,H,W], list of [K_b,7]."""
        ops.require_cuda()
        xh = x.permute(0, 2, 3, 1).contiguous()
        k_cap = max(1, max(len(g) for g in guided_anchors))
        dev = xh.device
        boxes = _pad_lists(guided_anchors, k_cap, 7, torch.float32, dev)
        d_k = torch.tensor([len(g) for g in guided_anchors], dtype=torch.int32, device=dev)
        scores = self.forward_device(xh, boxes, d_k)
        out = [scores[b, : len(g)] if len(g) else torch.empty(0, device=dev) for b, g in enumerate(guided_anchors)]
        return out if is_test else torch.cat(out, 0)

    def rescore_device(self, boxes, scores, labels, d_k, cfg, status):
        return ops.rescore_nms(boxes, scores, labels, d_k, float(cfg.score_thr), float(cfg.nms.iou_thr),
                               self.det_cap, status)

    def get_rescore_bboxes(self, guided_anchors, cls_scores, anchor_labels, img_metas, cfg):
        """Reference signature (ssd_rotate_head.py:487-533): lists in, lists of numpy arrays (or None) out."""
        ops.require_cuda()
        B = len(img_metas)
        dev = guided_anchors[0].device
        k_cap = max(1, max(len(g) for g in guided_anchors))
        boxes = _pad_lists([g.view(-1, 7) for g in guided_anchors], k_cap, 7, torch.float32, dev)
        scores = _pad_lists([s.view(-1) for s in cls_scores], k_cap, 0, torch.float32, dev)
        labels = _pad_lists(anchor_labels, k_cap, 0, torch.int32, dev)
        d_k = torch.tensor([len(g) for g in guided_anchors], dtype=torch.int32, device=dev)
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        det_cap = self.det_cap
        self.det_cap = max(self.det_cap, min(k_cap, ops.NMS_CAP))   # the reference applies no max_per_img
        try:
            det, d_ndet = self.rescore_device(boxes, scores, labels, d_k, cfg, status)
        finally:
            self.det_cap = det_cap
        return unpack_detections(det, d_ndet, status)


def unpack_detections(det, d_ndet, status=None):
    """Device [B,cap,9] + counts (+ the status word, checked) -> split_detections' three lists."""
    det_c = det.cpu().numpy()
    n = d_ndet.cpu().numpy()
    if status is not None:
        ops._lib.raise_on_status(status)
    return split_detections(det_c, n)


def split_detections(det, n):
    """Host [B,cap,9] rows + counts [B] -> the reference's three lists (numpy [D,7], [D], [D] or None)."""
    bbs, scs, lbs = [], [], []
    for b in range(det.shape[0]):
        k = int(n[b])
        if k == 0:
            bbs.append(None); scs.append(None); lbs.append(None)
            continue
        bbs.append(det[b, :k, :7].copy()); scs.append(det[b, :k, 7].copy())
        lbs.append(det[b, :k, 8].astype(np.int64))
    return bbs, scs, lbs

"""``mmdet.models.detectors`` mirror for the hot path: SingleStageDetector
(mmdet/models/detectors/single_stage.py:13-41,52-73,110-131; base.py:77-81).

Two entry points:
  * ``forward(img, img_meta, return_loss=False, **kwargs)`` / ``forward_test`` — the
    reference's call signature (tools/test.py:31) with pre-voxelized inputs produced by
    the dataset side (kitti.py:296-352);
  * ``forward_points(points)`` — the fused path from raw Velodyne points on the host:
    one H2D copy, voxelize + anchors_mask + backbone + neck + heads + PSWarp + NMS with
    every data-dependent size kept on the device, one D2H copy of the fixed-size result.
    With ``frustum_planes`` the frames are full sweeps, cropped to the camera frustum on the
    device first (the reference crops them offline into ``velodyne_reduced``); with ``image_fov`` they are raw-drive
    sweeps, cropped on the device to the points that project into the image (the reference's KittiVideo).  With ``metas``
    the step also formats its detections as KITTI annotations on the device (ops.kitti_format).  With
    ``point_outputs`` it also returns the auxiliary network's per-voxel foreground logits and centre offsets.
  * ``forward(..., return_loss=True)`` / ``forward_train`` and ``loss_points`` — the training losses, forward only, in
    eval() mode (csrc/targets.cu).  ``forward_points(..., gt_bboxes=, gt_labels=)`` and ``detect_stream(losses=True)``
    compute them in the detection step itself (validation losses beside the detections, eager or captured).
"""
import gc
import weakref

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from . import builder, ops
from .results import annos_from_rows, meta_block
from .single_stage_heads import gt_arrays, split_detections, stage_gt, unpack_detections

# The crop a step runs before voxelizing: the first element of a captured-graph key.  0 and 1 equal False and True, so
# a key reads (crop, kitti, point_outputs) with the frustum crop as True.  A step that also computes the losses has a
# fourth element, True; the other kinds keep their three-element keys.
CROP_NONE, CROP_FRUSTUM, CROP_IMAGE_FOV = 0, 1, 2


class SingleStageDetector(nn.Module):
    def __init__(self, backbone, neck=None, bbox_head=None, extra_head=None, train_cfg=None, test_cfg=None,
                 pretrained=None):
        super().__init__()
        self.backbone = builder.build_backbone(backbone)
        if neck is None:
            raise NotImplementedError
        self.neck = builder.build_neck(neck)
        if bbox_head is not None:
            self.rpn_head = builder.build_single_stage_head(bbox_head)
        if extra_head is not None:
            self.extra_head = builder.build_single_stage_head(extra_head)
        self.train_cfg = train_cfg
        self.test_cfg = test_cfg
        self.class_names = None          # set by the caller, tools/test.py:139
        self.guided_thr = 0.1            # hard-coded in the reference, single_stage.py:122
        self.voxel_generator = None      # fused path: attach_data_pipeline()
        self.anchor_set = None
        self._pinned = None
        self._mask_stream = None
        self._graphs = {}                 # (crop kind, kitti, point_outputs[, losses]) -> captured step (enable_cuda_graph)
        self._graph_args = None
        self._stream_slots = None
        self._stream_key = None
        self._sets = weakref.WeakSet()   # the DetectorSets this model is a member of (refresh_packed_weights)
        if isinstance(pretrained, str):
            from .checkpoint import load_params_from_file
            load_params_from_file(self, pretrained)
        self.eval()

    @property
    def with_rpn(self):
        return hasattr(self, "rpn_head") and self.rpn_head is not None

    def set_precision(self, precision, sparse=None):
        """ops.PREC_F16X3 (default) = Hopper tensor-core (wgmma) kernels on the fp32-accurate 3xFP16 operand split
        (TMA-fed dense convs, cp.async-fed sparse convs); ops.PREC_TF32X3 = the 3xTF32 tensor-core kernels;
        ops.PREC_FP32 = CUDA-core FFMA kernels (bisecting / accuracy yard-stick).  ``sparse`` optionally selects a
        different path for the 13 ruled sparse convs."""
        self.neck.set_precision(precision, sparse)
        self.rpn_head.precision = precision
        self.extra_head.precision = precision
        self.refresh_packed_weights()

    def refresh_packed_weights(self):
        """Called after parameters were (re)loaded (checkpoint.load_state_dict_into) or the precision changed.
        Captured steps bake in the device addresses of packed weights, folded BN vectors and layer constants and the
        kernel selection; eager use version-checks the packed / folded tensors, but a CUDA-graph replay never
        re-checks: drop every captured step (the single-step graphs of enable_cuda_graph and the detect_stream slots)
        so the next call re-captures."""
        self._graphs = {}
        self._stream_slots = None
        self._stream_key = None
        for s in list(self._sets):      # a DetectorSet's captured steps bake in this member's weights too
            s.refresh_packed_weights()

    # ------------------------------------------------------------------ reference-signature path
    def merge_second_batch(self, batch_args):
        """single_stage.py:52-73 (torch.cat / F.pad are data movement only)."""
        ret = {}
        for key, elems in batch_args.items():
            if key in ("voxels", "num_points"):
                ret[key] = torch.cat(elems, dim=0)
            elif key == "coordinates":
                ret[key] = torch.cat([F.pad(c, [1, 0, 0, 0], mode="constant", value=i)
                                      for i, c in enumerate(elems)], dim=0)
            elif key in ("img_meta", "gt_labels", "gt_bboxes", "gt_types"):
                ret[key] = elems
            elif isinstance(elems, dict):
                ret[key] = {k: torch.stack(v, dim=0) for k, v in elems.items()}
            else:
                ret[key] = torch.stack(elems, dim=0)
        return ret

    def forward(self, img=None, img_meta=None, return_loss=False, **kwargs):
        if return_loss:
            if self.training:
                raise NotImplementedError("the losses are computed forward only, with BatchNorm's running statistics: "
                                          "call .eval() first (training is not supported)")
            return self.forward_train(img, img_meta, **kwargs)
        return self.forward_test(img, img_meta, **kwargs)

    def forward_train(self, img, img_meta, **kwargs):
        """single_stage.py:75-108 for a model in eval() mode: the loss dict (aux_loss_cls, aux_loss_reg, rpn_loc_loss,
        rpn_cls_loss, rpn_dir_loss, loss_cls), each a [1] tensor, computed on the device without autograd.  kwargs as
        the training dataset gives them: voxels, num_points, coordinates, anchors / anchors_mask (per-class dicts or
        tensors), gt_bboxes (x, y, z_bottom, w, l, h, ry per frame), gt_labels, gt_types.  A frame without GT is all
        background (aux labels 0, masked anchors 0, no GT rows in the guided boxes); the reference never sees one."""
        ops.require_cuda()
        if self.training:
            raise NotImplementedError("forward_train runs in eval() mode only")
        if self.train_cfg is None:
            raise ValueError("forward_train needs train_cfg (build_from_config passes cfg.train_cfg)")
        batch_size = len(img_meta)
        dev = next(self.parameters()).device
        ret = self.merge_second_batch({k: v for k, v in kwargs.items() if v is not None})
        voxels = ret["voxels"].to(dev).float().contiguous()
        coords = ret["coordinates"].to(dev).int().contiguous()
        gt_bboxes = [torch.as_tensor(g).to(dev).float().reshape(-1, 7) for g in ret["gt_bboxes"]]
        gt_labels = [torch.as_tensor(g).to(dev).long().reshape(-1) for g in ret["gt_labels"]]
        anchors, anchors_mask = _on_device(ret["anchors"], dev), _on_device(ret["anchors_mask"], dev)
        vx = self.backbone(voxels, ret["num_points"].to(dev))
        x, conv6, point_misc = self.neck(vx, coords, batch_size, is_test=False)
        losses = dict()
        losses.update(self.neck.aux_loss(*point_misc, gt_bboxes=gt_bboxes))
        rpn_outs = self.rpn_head(x)
        losses.update(self.rpn_head.loss(*rpn_outs, gt_bboxes, gt_labels, ret.get("gt_types"), anchors, anchors_mask,
                                         self.train_cfg.rpn))
        guided_anchors, _ = self.rpn_head.get_guided_anchors(*rpn_outs, anchors, anchors_mask, gt_bboxes,
                                                             gt_labels, thr=self.train_cfg.rpn.anchor_thr)
        bbox_score = self.extra_head(conv6, guided_anchors)
        losses.update(self.extra_head.loss(bbox_score, gt_bboxes, gt_labels, guided_anchors, self.train_cfg.extra))
        return losses

    def forward_test(self, img, img_meta, **kwargs):
        """single_stage.py:110-131.  When every ``img_meta`` carries the KITTI calibration (``calib``) and the
        caller set ``class_names`` (tools/test.py:139) the return value is the reference's: the list of KITTI
        annotation dicts of ``kitti_bbox2results`` (transforms.py:225-279).  Without calibration (synthetic clouds)
        it returns, per frame, the inputs of that conversion: dict(boxes_lidar [D,7], scores [D], label_preds [D])."""
        ops.require_cuda()
        batch_size = len(img_meta)
        dev = next(self.parameters()).device
        ret = self.merge_second_batch({k: v for k, v in kwargs.items() if v is not None and k not in
                                       ("gt_labels", "gt_bboxes", "gt_types")})
        voxels = ret["voxels"].to(dev).float().contiguous()
        num_points = ret["num_points"].to(dev)
        coords = ret["coordinates"].to(dev).int().contiguous()
        vx = self.backbone(voxels, num_points)
        x, conv6 = self.neck(vx, coords, batch_size, is_test=True)
        rpn_outs = self.rpn_head.forward(x)
        guided_anchors, anchor_labels = self.rpn_head.get_guided_anchors(
            *rpn_outs, ret["anchors"].to(dev), ret["anchors_mask"].to(dev), None, None, thr=self.guided_thr)
        bbox_score = self.extra_head(conv6, guided_anchors, is_test=True)
        det_bboxes, det_scores, det_labels = self.extra_head.get_rescore_bboxes(
            guided_anchors, bbox_score, anchor_labels, img_meta, self.test_cfg.extra)
        if self.class_names is not None and all(isinstance(m, dict) and m.get("calib") is not None for m in img_meta):
            from .results import kitti_bbox2results
            return [kitti_bbox2results(b, s, l, m, class_names=self.class_names)
                    for b, s, l, m in zip(det_bboxes, det_scores, det_labels, img_meta)]
        return [dict(boxes_lidar=b, scores=s, label_preds=l) for b, s, l in zip(det_bboxes, det_scores, det_labels)]

    # ------------------------------------------------------------------ fused raw-points path
    def attach_data_pipeline(self, voxel_generator, anchor_set):
        """Give the detector the data-side objects of the config (cfg.data.val.generator /
        anchor_generator) so that raw points are the only per-frame input."""
        self.voxel_generator = voxel_generator
        dev = next(self.parameters()).device
        self.anchor_set = anchor_set.to(dev)
        return self

    def forward_device(self, points, pt_off, batch, max_points_per_frame, point_outputs=False, detections=True,
                       guided_thr=None):
        """Everything on the device, no synchronisation.  points [Ncap,4], pt_off [batch+1] int32.
        Returns (det [B,det_cap,9], d_ndet [B], status [1], aux dict); without ``detections`` the rescoring and NMS are
        skipped and det, d_ndet are None (the loss path reads only the guided boxes and their scores).  With ``point_outputs`` the aux dict also holds
        the auxiliary network's points_mean [cap,4] (b, x, y, z), point_cls [cap] and point_reg [cap,3] (neck.point_head)
        for the voxel rows (frame_rows).  ``guided_thr``: the guided anchors' score threshold (default self.guided_thr;
        the losses use train_cfg.rpn.anchor_thr)."""
        _require_batch(self, batch)
        status = torch.zeros((1,), dtype=torch.int32, device=points.device)
        vox = self.voxel_generator.generate_device(points, pt_off, batch, max_points_per_frame, status)
        return self.forward_voxels(vox, batch, status, point_outputs=point_outputs, detections=detections,
                                   guided_thr=guided_thr)

    def anchor_mask(self, coors, d_rows, batch):
        """The anchor mask [batch, Na] of the voxel coordinates, queued on a side stream (it only feeds the
        guided-anchor selection, so it runs next to the backbone).  Returns (mask, the stream to wait for)."""
        main = torch.cuda.current_stream()
        if self._mask_stream is None:
            self._mask_stream = torch.cuda.Stream(device=coors.device)
        self._mask_stream.wait_stream(main)
        with torch.cuda.stream(self._mask_stream):
            mask = self.anchor_set.mask_device(coors, d_rows, batch)
        return mask, self._mask_stream

    def forward_voxels(self, vox, batch, status, sparse_in=None, point_outputs=False, detections=True,
                       guided_thr=None, mask=None, neighbours=None):
        """forward_device from the voxelizer's outputs ``vox`` = generate_device's (voxels, coors, num_points, mean,
        frame_rows) on: the anchor mask, the sparse backbone, the BEV neck, the heads, PSWarp and the rescoring with
        NMS, on this model's weights.  ``sparse_in``: the level-0 sparse tensor with its rulebooks already queued
        (SpMiddleFHD.sparse_input over the same voxels), which the members of a DetectorSet share; without it the neck
        builds them.  ``mask``: anchor_mask's (mask, stream) over these voxels, which the checkpoints of a
        CheckpointSweep share; ``neighbours``: the auxiliary network's three_nn outputs (SpMiddleFHD.point_head)."""
        voxels, coors, num, mean, frame_rows = vox
        d_rows = frame_rows[batch:batch + 1]
        main = torch.cuda.current_stream()
        mask, mask_stream = self.anchor_mask(coors, d_rows, batch) if mask is None else mask
        out = self.neck.forward_nhwc(mean, coors, batch, d_rows=d_rows, status=status, point_outputs=point_outputs,
                                     sparse_in=sparse_in, neighbours=neighbours)
        y, conv6, xs = out[:3]
        main.wait_stream(mask_stream)
        head = self.rpn_head.forward_nhwc(y)
        anchors, _ = self.anchor_set.device_tensors()
        thr = self.guided_thr if guided_thr is None else guided_thr
        boxes, labels, index, d_k = self.rpn_head.guided_anchors_device(head, anchors, mask, thr, status)
        ps_feat = self.extra_head.convs_nhwc(conv6)
        scores = self.extra_head.sample(ps_feat, boxes, d_k)
        det = d_ndet = None
        if detections:
            det, d_ndet = self.extra_head.rescore_device(boxes, scores, labels, d_k, self.test_cfg.extra, status)
        aux = dict(voxels=voxels, coors=coors, num_points=num, mean=mean, frame_rows=frame_rows, mask=mask, x=y,
                   conv6=conv6, head=head, guided=boxes, guided_labels=labels, guided_index=index, d_k=d_k,
                   ps_feat=ps_feat, ps_scores=scores, sparse=xs)
        if point_outputs:
            aux.update(out[3])
        return det, d_ndet, status, aux

    def stage_points(self, points_list):
        """Host side of the fused path: concatenate the frames into one pinned buffer."""
        counts = [int(p.shape[0]) for p in points_list]
        total = sum(counts)
        need = max(total, 1)
        if self._pinned is None or self._pinned[0].shape[0] < need or self._pinned[1].shape[0] < len(counts) + 1:
            self._pinned = _pinned_pair(max(need, 1 << 16), max(len(counts) + 1, 65))
        hp, ho = self._pinned
        _stage_into(hp, ho, points_list, counts)
        return hp[:need], ho[:len(counts) + 1], counts

    # ------------------------------------------------------------------ CUDA-graph replay of the fused path
    def enable_cuda_graph(self, batch, max_points_per_frame=32768):
        """Capture forward_device once for (batch, max_points_per_frame) and replay it per step: every
        data-dependent size already lives on the device, so the ~65 launches of a step become one graph
        launch.  Steps whose shape does not fit fall back to the eager path.  forward_points replays one graph per kind
        of call: with ``frustum_planes``, with ``image_fov`` or without a crop (a cropping graph crops the full sweeps
        first, and ``max_points_per_frame`` bounds them, e.g. 131072), ``metas`` (it ends with the KITTI result
        formatter), ``point_outputs`` (it also runs the auxiliary network) and ``gt_bboxes`` (it also computes the
        losses).  The plain kind is captured here and returned, the others on their first use; a
        new call replaces every graph captured for an earlier shape."""
        self._graph_args = (int(batch), int(max_points_per_frame))
        self._graphs = {}
        return self._graph_for(CROP_NONE, False, False)

    def disable_cuda_graph(self):
        self._graphs = {}
        self._graph_args = None

    def _graph_for(self, crop, kitti, point_outputs, losses=False):
        """The captured single step of this kind at enable_cuda_graph's shape, captured on first use; None while the
        graphs are disabled."""
        key = (int(crop), kitti, point_outputs) + ((True,) if losses else ())
        if key not in self._graphs and self._graph_args is not None:
            self._graphs[key] = _GraphedStep(self, *self._graph_args, latency=True, crop=crop, kitti=kitti,
                                             point_outputs=point_outputs, losses=losses)
        return self._graphs.get(key)

    def _require_loss_step(self):
        """A detection step that also computes the losses needs train_cfg, eval() mode and one guided-anchor selection
        for both: train_cfg.rpn.anchor_thr must equal the test threshold (both shipped configs set 0.1)."""
        if self.training:
            raise NotImplementedError("the losses are computed in eval() mode only")
        if self.train_cfg is None:
            raise ValueError("the losses need train_cfg (build_from_config passes cfg.train_cfg)")
        thr = float(self.train_cfg.rpn.anchor_thr)
        if thr != self.guided_thr:
            raise ValueError("train_cfg.rpn.anchor_thr = %r differs from the test threshold %r: the losses and the "
                             "detections select different guided anchors, so one step cannot give both (use "
                             "loss_points)" % (thr, self.guided_thr))

    @staticmethod
    def _gt_inputs(gt_bboxes, gt_labels, batch):
        """Per-frame GT boxes and 1-based labels -> gt_arrays' (boxes, anchor classes = labels - 1, labels)."""
        if len(gt_bboxes) != batch or len(gt_labels) != batch:
            raise ValueError("one GT box set and label set per frame: %d frames, %d box sets, %d label sets" %
                             (batch, len(gt_bboxes), len(gt_labels)))
        labels = [np.asarray(l, np.int64).reshape(-1) for l in gt_labels]
        return gt_bboxes, [(l - 1).astype(np.int32) for l in labels], labels

    def detect_stream(self, batches, batch, max_points_per_frame=32768, depth=4, concurrent=True, crop=False,
                      kitti=False, image_fov=False, losses=False):
        """Throughput API: iterate over batches (each a list of ``batch`` raw point arrays) and yield their
        detections in order.  ``depth`` captured graphs with their own static buffers and scratch are used
        round-robin: while the GPU runs step i, the host stages and uploads step i+1 (copy stream) and unpacks
        step i-1.  With ``concurrent`` every slot replays on its own stream, so the low-occupancy phases of one
        step (voxelize, rulebooks, the sparse layers, NMS) run beside the dense layers of its neighbour.
        With ``crop`` each item of ``batches`` is (points_list, planes [batch,6,4]) of full sweeps: every slot's graph
        crops the frames to their camera frustums (forward_points' ``frustum_planes``) before the step, and
        ``max_points_per_frame`` bounds the full sweeps.
        With ``kitti`` each item also carries the frames' ``img_meta``-style dicts (forward_points' ``metas``):
        (points_list, planes, metas) with ``crop``, else (points_list, metas); every slot's graph ends with the KITTI
        result formatter and each yield is the batch's annotation dicts (kitti_bbox2results' format).
        With ``image_fov`` (needs ``kitti``, excludes ``crop``) the items are (points_list, metas) of raw-drive sweeps:
        every slot's graph first crops each frame to the points that project into its image (forward_points'
        ``image_fov``).
        With ``losses`` each item ends with the batch's ground truth, (gt_bboxes, gt_labels) as forward_points takes
        them: every slot's graph also computes the losses, and each yield is (results, losses), ``losses`` the batch's
        dict of floats (loss_points')."""
        ops.require_cuda()
        if kitti and self.class_names is None:
            raise ValueError("detect_stream(kitti=True) needs class_names")
        kind = _crop_kind(bool(crop), image_fov, kitti)
        losses = bool(losses)
        if losses:
            self._require_loss_step()
        key = (batch, max_points_per_frame, depth, kind, bool(kitti), losses)
        if self._stream_key != key or self._stream_slots is None:
            self._stream_slots = [_GraphedStep(self, batch, max_points_per_frame, crop=kind, kitti=kitti, losses=losses)
                                  for _ in range(depth)]
            self._copy_stream = torch.cuda.Stream()
            self._stream_key = key
        yield from _stream_through(self, batches, batch, max_points_per_frame, depth, concurrent, crop, kitti, losses)

    def _collected(self, slot, metas):
        """Wait for a slot's step and convert its host copy into the caller's per-frame results (and its losses)."""
        res = self._frame_results(slot.collect(), metas)
        return (res, slot.loss_results()) if slot.losses else res

    def _frame_results(self, out, metas):
        """A step's host outputs -> the caller's per-frame results: with ``metas`` KITTI annotation dicts of the
        formatter's (rows, n_out), else detection dicts of split_detections' (boxes, scores, labels)."""
        if metas is not None:
            return annos_from_rows(*out, self.class_names, [m["sample_idx"] for m in metas])
        return [dict(boxes_lidar=b, scores=s, label_preds=l) for b, s, l in zip(*out)]

    def forward_points(self, points_list, return_aux=False, frustum_planes=None, metas=None, point_outputs=False,
                       image_fov=False, gt_bboxes=None, gt_labels=None):
        """Raw points in (list of [N_i,>=4] numpy arrays), detections out: per frame a dict of
        boxes_lidar [D,7], scores [D], label_preds [D] (or None entries when nothing survives).
        ``frustum_planes``: one float64 [6,4] array per frame (frustum.camera_frustum_planes).  The frames are then
        full sweeps; each is cropped to its camera frustum on the device, in point order (ops.frustum_crop), and the
        step runs on what is left, as on the reference's offline-cropped ``velodyne_reduced`` clouds.
        ``metas``: one ``img_meta``-style dict per frame ('calib' a results.Calibration, 'img_shape', 'sample_idx').
        The detections are then formatted on the device (ops.kitti_format) and the call returns, like forward_test,
        one KITTI annotation dict per frame; ``class_names`` must be set.  With ``return_aux`` the aux dict also holds
        the unformatted detections (det, ndet).
        ``point_outputs``: the step also runs SA-SSD's auxiliary network (neck.point_head) and the call returns
        (results, points), results as without it and ``points`` one dict per frame of xyz [V,3] (the voxel means),
        cls [V] (foreground logits) and reg [V,3] (offsets to the box centre), V the frame's voxels in voxel-row order.
        With ``return_aux`` the aux dict comes third.
        ``image_fov``: the frames are raw-drive sweeps; each is cropped on the device, in point order, to the points
        that project into its image and lie in front of x = 0.1 m (ops.image_fov_crop), as the reference's KittiVideo
        crops them (get_lidar_in_image_fov).  Needs ``metas``, whose calibration and image shape define the crop, and
        excludes ``frustum_planes``.
        ``gt_bboxes`` / ``gt_labels``: per frame the GT boxes [G,7] and 1-based labels as loss_points takes them.  The
        same step then also computes SA-SSD's losses (loss_device, after the detections and before the formatter) and
        the call returns (results, losses), ``results`` exactly as without GT and ``losses`` loss_points' dict of
        floats for these frames; with ``point_outputs`` the points come before the losses, with ``return_aux`` the aux
        dict last.  Needs train_cfg with rpn.anchor_thr equal to the test threshold (one guided-anchor selection
        serves both); a frame with more than SASSD_GT_CAP_MAX boxes raises."""
        ops.require_cuda()
        if self.voxel_generator is None or self.anchor_set is None:
            raise RuntimeError("call attach_data_pipeline(voxel_generator, anchor_set) first")
        if metas is not None and self.class_names is None:
            raise ValueError("forward_points(metas=) needs class_names")
        kind = _crop_kind(frustum_planes is not None, image_fov, metas is not None)
        B = len(points_list)
        losses = gt_bboxes is not None or gt_labels is not None
        gt_in = None
        if losses:
            self._require_loss_step()
            if gt_bboxes is None or gt_labels is None:
                raise ValueError("forward_points: gt_bboxes and gt_labels go together")
            gt_in = self._gt_inputs(gt_bboxes, gt_labels, B)
        planes = None if frustum_planes is None else _frame_planes(frustum_planes, B)
        meta = None if metas is None else _meta_blocks(metas, B)
        hp, ho, counts = self.stage_points(points_list)
        g = self._graph_for(kind, meta is not None, bool(point_outputs), losses)
        if g is not None and not return_aux and g.fits(B, counts):
            res = self._frame_results(g.run_host(hp, ho, sum(counts), planes, meta, gt_in), metas)
            ret = (res,) + ((g.point_results(),) if point_outputs else ()) + ((g.loss_results(),) if losses else ())
            return ret if len(ret) > 1 else res
        dev = next(self.parameters()).device
        gt = stage_gt(*gt_in, dev) if losses else None
        det, d_ndet, status, aux = _run_step(self, hp.to(dev, non_blocking=True), ho.to(dev, non_blocking=True), B,
                                             max(counts + [1]), _to_device(planes, dev), _to_device(meta, dev),
                                             point_outputs=point_outputs, image_fov=kind == CROP_IMAGE_FOV, gt=gt)
        if meta is not None:
            ops._lib.raise_on_status(status)
            out = aux["rows"].cpu().numpy(), aux["n_out"].cpu().numpy()
            aux.update(det=det, ndet=d_ndet)
        else:
            out = unpack_detections(det, d_ndet, status)
        res = self._frame_results(out, metas)
        pts = _split_points(*(aux[k].cpu().numpy() for k in _POINT_KEYS)) if point_outputs else None
        loss = _loss_dict(aux["losses"].cpu()) if losses else None
        ret = (res,) + ((pts,) if point_outputs else ()) + ((loss,) if losses else ()) + ((aux,) if return_aux else ())
        return ret if len(ret) > 1 else res

    def loss_targets(self, aux, batch, gt, gt_class, gt_label, d_ngt, status):
        """The targets of loss_device that read coordinates, anchors, the anchor mask and GT only, no prediction:
        (points_in_boxes' (labels, offsets, d_npos) of the voxel means, SSDRotateHead.assign's (labels, targets, ious,
        d_npos)).  The checkpoints of a CheckpointSweep share them."""
        d_rows = aux["frame_rows"][batch:batch + 1]
        points = ops.points_in_boxes(aux["points_mean"], d_rows, gt, d_ngt, status)
        return points, self._assign_rpn(aux, gt, gt_class, gt_label, d_ngt, status)

    def _assign_rpn(self, aux, gt, gt_class, gt_label, d_ngt, status):
        anchors, _ = self.anchor_set.device_tensors()
        names = list(self.class_names) if self.class_names is not None else [None]
        pos, neg = self.rpn_head.thresholds(self.train_cfg.rpn, names)
        return self.rpn_head.assign(anchors, aux["mask"], gt, gt_class, gt_label, d_ngt, pos, neg, status)

    def loss_device(self, aux, batch, gt, gt_class, gt_label, d_ngt, n_gt_host, status, targets=None):
        """Targets and losses of one forward_device(point_outputs=True) step, on the device: returns the loss vector
        [6] in ops.LOSS_KEYS order and a dict of the targets.  gt [B,gt_cap,7] etc. as stage_gt gives them.  Nothing
        here reads the host: PSWarp scores min(d_ngt[b], gt_cap) GT rows of each frame, the cap applied by the pswarp
        and assign_pswarp kernels, so the step can be captured; ``n_gt_host`` is not read.  ``targets``: loss_targets'
        outputs for this step's voxels, anchor mask and GT, which are then not computed again."""
        dev = gt.device
        gt_cap = gt.shape[1]
        out = torch.zeros((len(ops.LOSS_KEYS),), dtype=torch.float32, device=dev)
        cfg = self.train_cfg
        d_rows = aux["frame_rows"][batch:batch + 1]
        if targets is None:
            p_lab, p_off, p_npos = ops.points_in_boxes(aux["points_mean"], d_rows, gt, d_ngt, status)
        else:
            (p_lab, p_off, p_npos), rpn = targets
        ops.aux_loss(aux["point_cls"], aux["point_reg"], p_lab, p_off, d_rows, batch, p_npos, out[0:2])
        if targets is None:
            rpn = self._assign_rpn(aux, gt, gt_class, gt_label, d_ngt, status)
        anchors, _ = self.anchor_set.device_tensors()
        r_lab, r_tgt, r_iou, _ = self.rpn_head.loss_device(aux["head"], anchors, aux["mask"], gt, gt_class, gt_label,
                                                           d_ngt, pos_thr=None, neg_thr=None, out=out[2:5],
                                                           status=status, targets=rpn)
        # PSWarp scores the GT rows the reference prepends to each frame's guided boxes (:364-367) in a slot segment of
        # their own, so the guided capacity does not grow
        gt_scores = self.extra_head.sample(aux["ps_feat"], gt, d_ngt)
        boxes = torch.cat([gt, aux["guided"]], 1).contiguous()
        scores = torch.cat([gt_scores, aux["ps_scores"]], 1).contiguous()
        e_lab, e_iou, _ = self.extra_head.loss_device(scores, boxes, aux["d_k"], gt, d_ngt, cfg.extra, out[5:6], status,
                                                      d_head=d_ngt, head_cap=gt_cap)
        return out, dict(point_labels=p_lab, point_offsets=p_off, rpn_labels=r_lab, rpn_targets=r_tgt, rpn_ious=r_iou,
                         ps_boxes=boxes, ps_scores=scores, ps_labels=e_lab, ps_ious=e_iou)

    def loss_points(self, points_list, gt_bboxes, gt_labels, frustum_planes=None, return_aux=False):
        """The losses of forward(return_loss=True) from raw points: ``points_list`` as forward_points takes it, per frame
        the GT boxes [G,7] (x, y, z_bottom, w, l, h, ry, lidar frame) and their labels (1-based over class_names; a box
        counts for the anchors of class_names[label - 1]).  Runs forward_device(point_outputs=True) up to the guided boxes'
        PSWarp scores (no rescoring or NMS), scores the GT boxes
        on PSWarp's map, then every target and loss on the device; one device-to-host copy of the loss vector and the
        status word.  Returns a dict of Python floats keyed like forward_train (with ``return_aux`` also the step's aux
        dict and the targets).  The model must be in eval() mode; frames without GT are all background."""
        ops.require_cuda()
        if self.training:
            raise NotImplementedError("loss_points runs in eval() mode only")
        if self.voxel_generator is None or self.anchor_set is None:
            raise RuntimeError("call attach_data_pipeline(voxel_generator, anchor_set) first")
        if self.train_cfg is None:
            raise ValueError("loss_points needs train_cfg (build_from_config passes cfg.train_cfg)")
        B = len(points_list)
        gt_in = self._gt_inputs(gt_bboxes, gt_labels, B)
        dev = next(self.parameters()).device
        planes = None if frustum_planes is None else _frame_planes(frustum_planes, B)
        hp, ho, counts = self.stage_points(points_list)
        _, _, status, aux = _run_step(self, hp.to(dev, non_blocking=True), ho.to(dev, non_blocking=True), B,
                                      max(counts + [1]), _to_device(planes, dev), detections=False,
                                      guided_thr=float(self.train_cfg.rpn.anchor_thr), gt=stage_gt(*gt_in, dev))
        h = torch.empty((len(ops.LOSS_KEYS) + 1,), dtype=torch.float32, pin_memory=True)
        h[:-1].copy_(aux["losses"], non_blocking=True)
        h[-1:].copy_(status.view(torch.float32), non_blocking=True)
        torch.cuda.current_stream().synchronize()
        ops._lib.raise_on_status(h[-1:].view(torch.int32))
        res = _loss_dict(h[:-1])
        targets = aux.pop("targets")
        if return_aux:
            aux.update(targets)
            return res, aux
        return res


class DetectorSet:
    """Several single-class detectors run as one: each KITTI class by a model of its own, as the reference's single-class
    checkpoints are meant to be used, in one step over shared inputs.

    ``models``: built SingleStageDetectors in eval() mode, each with its class names and data pipeline attached
    (build_from_config).  They must share the voxel grid - the voxel generator's voxel size, point-cloud range,
    max_num_points and max_voxels - the neck's output_shape and its row_cap_factor (the rulebooks' capacities), and no
    class may belong to two members (ValueError otherwise).  Member 0's neck builds the shared rulebooks, so its
    overlap_rulebooks setting (side streams or not; the rulebooks are the same) applies to the whole set.  The set's class list is the members' class names concatenated in member order, and the
    labels it returns index that list.

    One step crops (when asked), copies, voxelizes and builds the seven rulebooks once, then runs each member's anchor
    mask, sparse backbone, BEV neck, heads, PSWarp and rescoring with NMS on its own weights, and gathers the members'
    detections per frame in member order (ops.merge_detections).  There is no NMS across members: each frame's
    detections are exactly the concatenation of what each member's forward_points returns for it, and with ``metas`` its
    KITTI rows are the concatenation of the members' rows.  A set of one model returns what that model returns.

    forward_points, enable_cuda_graph and detect_stream take the items and return the results of the
    SingleStageDetector methods of the same names (without losses, auxiliary outputs or return_aux).  The set keeps
    its own captured graphs and stream slots; the members' own are neither used nor changed.  Loading parameters into
    a member or changing its precision (refresh_packed_weights) drops the set's captured steps too."""

    def __init__(self, models):
        models = list(models)
        if not models:
            raise ValueError("a DetectorSet needs at least one model")
        if len(models) > ops._lib.MERGE_MAX:
            raise ValueError("a DetectorSet takes at most %d models, got %d" % (ops._lib.MERGE_MAX, len(models)))
        for i, m in enumerate(models):
            if not isinstance(m, SingleStageDetector):
                raise TypeError("member %d is a %s, not a SingleStageDetector" % (i, type(m).__name__))
            if m.training:
                raise ValueError("member %d is in training mode: call .eval() first" % i)
            if m.voxel_generator is None or m.anchor_set is None or m.class_names is None:
                raise ValueError("member %d has no data pipeline or class names (build_from_config attaches them)" % i)
        lead = models[0]
        for i, m in enumerate(models[1:], 1):
            diff = voxel_grid_difference(lead.voxel_generator, m.voxel_generator)
            if diff:
                raise ValueError("member %d voxelizes differently from member 0 (%s): the set shares one voxelizer "
                                 "and one set of rulebooks, so run such models separately" % (i, diff))
            if list(m.neck.sparse_shape) != list(lead.neck.sparse_shape):
                raise ValueError("member %d's neck output_shape %s differs from member 0's %s" %
                                 (i, list(m.neck.sparse_shape), list(lead.neck.sparse_shape)))
            if m.neck.row_cap_factor != lead.neck.row_cap_factor:
                raise ValueError("member %d's neck row_cap_factor %r differs from member 0's %r: the shared rulebooks "
                                 "have one set of capacities" % (i, m.neck.row_cap_factor, lead.neck.row_cap_factor))
            if next(m.parameters()).device != next(lead.parameters()).device:
                raise ValueError("member %d is on another device than member 0" % i)
        self.models = models
        self.class_names, self.label_offsets = merged_classes([m.class_names for m in models])
        self._pinned = None
        self._graphs = {}                 # (crop kind, kitti) -> the set's captured step (enable_cuda_graph)
        self._graph_args = None
        self._stream_slots = None
        self._stream_key = None
        for m in models:
            m._sets.add(self)

    def parameters(self):
        for m in self.models:
            yield from m.parameters()

    @property
    def det_cap(self):
        """Detection rows per frame of the merged block: the members' capacities summed."""
        return sum(m.extra_head.det_cap for m in self.models)

    def refresh_packed_weights(self):
        """Drop every captured step of the set (a member's parameters or precision changed)."""
        self._graphs = {}
        self._stream_slots = None
        self._stream_key = None

    stage_points = SingleStageDetector.stage_points
    disable_cuda_graph = SingleStageDetector.disable_cuda_graph
    _frame_results = SingleStageDetector._frame_results
    _collected = SingleStageDetector._collected

    def enable_cuda_graph(self, batch, max_points_per_frame=32768):
        """SingleStageDetector.enable_cuda_graph for the set's step: the plain kind is captured here and returned,
        the crop and KITTI kinds on their first use."""
        self._graph_args = (int(batch), int(max_points_per_frame))
        self._graphs = {}
        return self._graph_for(CROP_NONE, False)

    def _graph_for(self, crop, kitti):
        key = (int(crop), kitti)
        if key not in self._graphs and self._graph_args is not None:
            self._graphs[key] = _GraphedStep(self, *self._graph_args, latency=True, crop=crop, kitti=kitti,
                                             run_step=_set_step)
        return self._graphs.get(key)

    def forward_points(self, points_list, frustum_planes=None, metas=None, image_fov=False):
        """SingleStageDetector.forward_points for the set: per frame a dict of boxes_lidar, scores and label_preds
        (None entries when no member keeps a box), or with ``metas`` one KITTI annotation dict, each holding every
        member's detections in member order."""
        ops.require_cuda()
        kind = _crop_kind(frustum_planes is not None, image_fov, metas is not None)
        B = len(points_list)
        planes = None if frustum_planes is None else _frame_planes(frustum_planes, B)
        meta = None if metas is None else _meta_blocks(metas, B)
        hp, ho, counts = self.stage_points(points_list)
        g = self._graph_for(kind, meta is not None)
        if g is not None and g.fits(B, counts):
            return self._frame_results(g.run_host(hp, ho, sum(counts), planes, meta), metas)
        dev = next(self.parameters()).device
        det, d_ndet, status, aux = _set_step(self, hp.to(dev, non_blocking=True), ho.to(dev, non_blocking=True), B,
                                             max(counts + [1]), _to_device(planes, dev), _to_device(meta, dev),
                                             image_fov=kind == CROP_IMAGE_FOV)
        if meta is not None:
            ops._lib.raise_on_status(status)
            out = aux["rows"].cpu().numpy(), aux["n_out"].cpu().numpy()
        else:
            out = unpack_detections(det, d_ndet, status)
        return self._frame_results(out, metas)

    def detect_stream(self, batches, batch, max_points_per_frame=32768, depth=4, concurrent=True, crop=False,
                      kitti=False, image_fov=False):
        """SingleStageDetector.detect_stream for the set: the same items, ``depth`` captured set steps used
        round-robin, and per batch the merged results of forward_points."""
        ops.require_cuda()
        kind = _crop_kind(bool(crop), image_fov, kitti)
        key = (batch, max_points_per_frame, depth, kind, bool(kitti))
        if self._stream_key != key or self._stream_slots is None:
            self._stream_slots = [_GraphedStep(self, batch, max_points_per_frame, crop=kind, kitti=kitti,
                                               run_step=_set_step) for _ in range(depth)]
            self._copy_stream = torch.cuda.Stream()
            self._stream_key = key
        yield from _stream_through(self, batches, batch, max_points_per_frame, depth, concurrent, crop, kitti, False)


class CheckpointSweep:
    """Several checkpoints of one config validated as one: the same frames, the same step, each checkpoint's detections
    and losses.  This is how a training run's saved checkpoints are compared on a labelled split.

    ``models``: K >= 1 SingleStageDetectors built from one config (build_from_config), each with its own weights, in
    eval() mode and on one device.  They must share the voxel grid, the neck's output_shape and row_cap_factor, the
    anchors, class_names, train_cfg, test_cfg and the detection capacity (ValueError otherwise): the step computes
    everything that depends on these and not on the weights once.

    One step crops (when asked), copies, voxelizes, builds the seven rulebooks and the anchor mask once; with GT it
    also computes the auxiliary network's nearest voxel centres (three_nn), the point targets (points_in_boxes) and
    the RPN targets (assign_rpn) once.  Per checkpoint it runs the sparse backbone, BEV neck, heads, PSWarp, rescoring
    and NMS, the auxiliary head, the PSWarp targets and the loss reductions, and with ``metas`` the KITTI formatter on
    that checkpoint's block.  The checkpoints share one status word, checked when the step's results are read.

    forward_points, enable_cuda_graph and detect_stream take the items of the SingleStageDetector methods of the same
    names (losses included; without auxiliary outputs or return_aux) and return a list of K results in member order:
    entry k is exactly what member k returns for the same call.  A sweep of one model returns [that model's result].
    The sweep keeps its own captured graphs and stream slots; reloading a member's parameters or changing its
    precision drops them.

    Memory: one step holds the front end and one network's activations at a time (each member's are freed before the
    next runs), so a captured step's graph pool hardly grows with K.  On an H100 80GB HBM3 at batch 16 of full sweeps
    with the losses it measured 7.9 GB at K = 4 and at K = 10, against 7.2 GB for one model
    (tests/tools/checkpoint_sweep_memory.py); each checkpoint's weights and cached empty-scene maps add about 0.33 GB.
    detect_stream's ``depth`` slots each hold one such step: test.py's four take about 32 GB at batch 16."""

    def __init__(self, models):
        models = list(models)
        if not models:
            raise ValueError("a CheckpointSweep needs at least one model")
        for i, m in enumerate(models):
            if not isinstance(m, SingleStageDetector):
                raise TypeError("member %d is a %s, not a SingleStageDetector" % (i, type(m).__name__))
            if m.training:
                raise ValueError("member %d is in training mode: call .eval() first" % i)
            if m.voxel_generator is None or m.anchor_set is None or m.class_names is None:
                raise ValueError("member %d has no data pipeline or class names (build_from_config attaches them)" % i)
        lead = models[0]
        for i, m in enumerate(models[1:], 1):
            diff = config_difference(lead, m)
            if diff:
                raise ValueError("member %d differs from member 0 in %s: a sweep compares checkpoints of one config" %
                                 (i, diff))
            if next(m.parameters()).device != next(lead.parameters()).device:
                raise ValueError("member %d is on another device than member 0" % i)
        self.models = models
        self.class_names = list(lead.class_names)
        self._pinned = None
        self._graphs = {}                 # (crop kind, kitti, losses) -> the sweep's captured step (enable_cuda_graph)
        self._graph_args = None
        self._stream_slots = None
        self._stream_key = None
        for m in models:
            m._sets.add(self)

    parameters = DetectorSet.parameters
    refresh_packed_weights = DetectorSet.refresh_packed_weights
    stage_points = SingleStageDetector.stage_points
    disable_cuda_graph = SingleStageDetector.disable_cuda_graph
    _gt_inputs = staticmethod(SingleStageDetector._gt_inputs)

    def _require_loss_step(self):
        for m in self.models:
            m._require_loss_step()

    def enable_cuda_graph(self, batch, max_points_per_frame=32768):
        """SingleStageDetector.enable_cuda_graph for the sweep's step: the plain kind is captured here and returned,
        the crop, KITTI and loss kinds on their first use."""
        self._graph_args = (int(batch), int(max_points_per_frame))
        self._graphs = {}
        return self._graph_for(CROP_NONE, False)

    def _graph_for(self, crop, kitti, losses=False):
        key = (int(crop), kitti, losses)
        if key not in self._graphs and self._graph_args is not None:
            self._graphs[key] = _GraphedStep(self, *self._graph_args, latency=True, crop=crop, kitti=kitti,
                                             losses=losses, run_step=_sweep_step)
        return self._graphs.get(key)

    def _frame_results(self, out, metas):
        """A step's host outputs, the K members' blocks one after another -> per member the frame results of
        SingleStageDetector._frame_results."""
        K = len(self.models)
        if metas is not None:
            res = annos_from_rows(*out, self.class_names, [m["sample_idx"] for m in metas] * K)
        else:
            res = [dict(boxes_lidar=b, scores=s, label_preds=l) for b, s, l in zip(*out)]
        B = len(res) // K
        return [res[k * B:(k + 1) * B] for k in range(K)]

    def _loss_results(self, h):
        """The K members' loss vectors, one after another -> one dict of floats per member."""
        n = len(ops.LOSS_KEYS)
        return [_loss_dict(h[k * n:(k + 1) * n]) for k in range(len(self.models))]

    def _collected(self, slot, metas):
        res = self._frame_results(slot.collect(), metas)
        return list(zip(res, self._loss_results(slot.h_loss))) if slot.losses else res

    def forward_points(self, points_list, frustum_planes=None, metas=None, image_fov=False, gt_bboxes=None,
                       gt_labels=None):
        """SingleStageDetector.forward_points for every member in one step: a list with, per member, what its own
        forward_points returns for these arguments ((results, losses) with GT)."""
        ops.require_cuda()
        kind = _crop_kind(frustum_planes is not None, image_fov, metas is not None)
        B = len(points_list)
        losses = gt_bboxes is not None or gt_labels is not None
        gt_in = None
        if losses:
            self._require_loss_step()
            if gt_bboxes is None or gt_labels is None:
                raise ValueError("forward_points: gt_bboxes and gt_labels go together")
            gt_in = self._gt_inputs(gt_bboxes, gt_labels, B)
        planes = None if frustum_planes is None else _frame_planes(frustum_planes, B)
        meta = None if metas is None else _meta_blocks(metas, B)
        hp, ho, counts = self.stage_points(points_list)
        g = self._graph_for(kind, meta is not None, losses)
        if g is not None and g.fits(B, counts):
            res = self._frame_results(g.run_host(hp, ho, sum(counts), planes, meta, gt_in), metas)
            return list(zip(res, self._loss_results(g.h_loss))) if losses else res
        dev = next(self.parameters()).device
        gt = stage_gt(*gt_in, dev) if losses else None
        det, d_ndet, status, aux = _sweep_step(self, hp.to(dev, non_blocking=True), ho.to(dev, non_blocking=True), B,
                                               max(counts + [1]), _to_device(planes, dev), _to_device(meta, dev),
                                               image_fov=kind == CROP_IMAGE_FOV, gt=gt)
        if meta is not None:
            ops._lib.raise_on_status(status)
            out = aux["rows"].cpu().numpy(), aux["n_out"].cpu().numpy()
        else:
            out = unpack_detections(det, d_ndet, status)
        res = self._frame_results(out, metas)
        return list(zip(res, self._loss_results(aux["losses"].cpu()))) if losses else res

    def detect_stream(self, batches, batch, max_points_per_frame=32768, depth=4, concurrent=True, crop=False,
                      kitti=False, image_fov=False, losses=False):
        """SingleStageDetector.detect_stream for the sweep: the same items, ``depth`` captured sweep steps used
        round-robin, and per batch a list with each member's yield."""
        ops.require_cuda()
        kind = _crop_kind(bool(crop), image_fov, kitti)
        losses = bool(losses)
        if losses:
            self._require_loss_step()
        key = (batch, max_points_per_frame, depth, kind, bool(kitti), losses)
        if self._stream_key != key or self._stream_slots is None:
            self._stream_slots = [_GraphedStep(self, batch, max_points_per_frame, crop=kind, kitti=kitti, losses=losses,
                                               run_step=_sweep_step) for _ in range(depth)]
            self._copy_stream = torch.cuda.Stream()
            self._stream_key = key
        yield from _stream_through(self, batches, batch, max_points_per_frame, depth, concurrent, crop, kitti, losses)


def config_difference(a, b):
    """What differs between two SingleStageDetectors in what a CheckpointSweep computes once for all of its members
    ('' when nothing): the voxel grid, the neck's output_shape and row_cap_factor, the anchors, class_names,
    train_cfg, test_cfg, the detection capacity."""
    diff = []
    grid = voxel_grid_difference(a.voxel_generator, b.voxel_generator)
    if grid:
        diff.append("voxel grid (%s)" % grid)
    if list(a.neck.sparse_shape) != list(b.neck.sparse_shape):
        diff.append("neck output_shape %s vs %s" % (list(a.neck.sparse_shape), list(b.neck.sparse_shape)))
    if a.neck.row_cap_factor != b.neck.row_cap_factor:
        diff.append("neck row_cap_factor %r vs %r" % (a.neck.row_cap_factor, b.neck.row_cap_factor))
    sa, sb = a.anchor_set, b.anchor_set
    if not (np.array_equal(sa.anchors, sb.anchors) and np.array_equal(sa.rects, sb.rects)
            and sa.grid_hw == sb.grid_hw and sa.threshold == sb.threshold):
        diff.append("anchors")
    if list(a.class_names) != list(b.class_names):
        diff.append("class_names %s vs %s" % (list(a.class_names), list(b.class_names)))
    if a.train_cfg != b.train_cfg:
        diff.append("train_cfg")
    if a.test_cfg != b.test_cfg:
        diff.append("test_cfg")
    if a.extra_head.det_cap != b.extra_head.det_cap:
        diff.append("detection capacity %d vs %d" % (a.extra_head.det_cap, b.extra_head.det_cap))
    return ", ".join(diff)


def merged_classes(class_lists):
    """The class list of a DetectorSet and each member's label offset into it: the members' class names
    concatenated in member order, member m's labels shifted by the number of classes before it.  A class in two
    members raises ValueError."""
    names, offsets = [], []
    for names_m in class_lists:
        offsets.append(len(names))
        names += list(names_m)
    dup = sorted({n for n in names if names.count(n) > 1})
    if dup:
        raise ValueError("class %s belongs to more than one member: a set keeps one model per class" % ", ".join(dup))
    return names, offsets


def voxel_grid_difference(a, b):
    """What differs between two VoxelGenerators' voxel grids ('' when nothing): voxel size, point-cloud range,
    max_num_points, max_voxels."""
    diff = []
    if not np.array_equal(a.voxel_size, b.voxel_size):
        diff.append("voxel size %s vs %s" % (list(a.voxel_size), list(b.voxel_size)))
    if not np.array_equal(a.point_cloud_range, b.point_cloud_range):
        diff.append("point-cloud range %s vs %s" % (list(a.point_cloud_range), list(b.point_cloud_range)))
    if a.max_num_points_per_voxel != b.max_num_points_per_voxel:
        diff.append("max_num_points %d vs %d" % (a.max_num_points_per_voxel, b.max_num_points_per_voxel))
    if a.max_voxels != b.max_voxels:
        diff.append("max_voxels %d vs %d" % (a.max_voxels, b.max_voxels))
    return ", ".join(diff)


def _on_device(v, dev):
    """A tensor or a per-class dict of tensors, on ``dev``."""
    return {k: t.to(dev) for k, t in v.items()} if isinstance(v, dict) else v.to(dev)


_POINT_KEYS = ("points_mean", "point_cls", "point_reg", "frame_rows")     # the aux outputs _split_points takes


def _split_points(points_mean, cls, reg, frame_rows):
    """Capacity-sized aux outputs (host) -> one dict per frame of its voxel rows: xyz [V,3], cls [V], reg [V,3]."""
    out = []
    for b in range(frame_rows.shape[0] - 1):
        r0, r1 = int(frame_rows[b]), int(frame_rows[b + 1])
        out.append(dict(xyz=points_mean[r0:r1, 1:4].copy(), cls=cls[r0:r1].copy(), reg=reg[r0:r1].copy()))
    return out


def _crop_kind(frustum, image_fov, kitti):
    """The crop kind of a step from its arguments; the image-FOV crop reads the frames' meta blocks, so it needs them."""
    if image_fov and frustum:
        raise ValueError("image_fov and a frustum crop exclude each other: a frame is cropped once")
    if image_fov and not kitti:
        raise ValueError("image_fov needs metas (kitti=True for detect_stream): the crop reads each frame's calibration "
                         "and image shape")
    return CROP_IMAGE_FOV if image_fov else CROP_FRUSTUM if frustum else CROP_NONE


def _frame_planes(frustum_planes, batch):
    """One [6,4] plane set per frame -> contiguous float64 [batch,6,4]."""
    planes = np.ascontiguousarray(np.asarray(frustum_planes, dtype=np.float64))
    if planes.shape != (batch, 6, 4):
        raise ValueError("frustum_planes: expected %d arrays of shape [6,4], got shape %s" % (batch, planes.shape))
    return planes


def _meta_blocks(metas, batch):
    """One ``img_meta``-style dict per frame -> contiguous float64 [batch,36] (results.meta_block)."""
    if len(metas) != batch:
        raise ValueError("metas: expected %d dicts, got %d" % (batch, len(metas)))
    return np.stack([meta_block(m["calib"], m["img_shape"]) for m in metas])


def _to_device(a, dev):
    """A host numpy array (or None) -> a tensor on ``dev``."""
    return None if a is None else torch.from_numpy(a).to(dev)


def _loss_dict(h):
    """A host loss vector [6] (ops.LOSS_KEYS order) -> dict of Python floats."""
    return {k: float(v) for k, v in zip(ops.LOSS_KEYS, h.tolist())}


def _require_batch(model, batch):
    """Refuse a step of more frames than the level-0 hash can key before any of its kernels is launched (the hash
    build would refuse it midway, after the voxelizer and the anchor mask ran)."""
    limit = model.neck.max_batch()
    if batch > limit:
        grid = "x".join(map(str, model.neck.sparse_shape))
        raise ops._lib.SassdError("batch %d exceeds the level-0 hash limit of %d frames: its 31-bit keys flatten "
                                  "(b, z, y, x) over the %s grid" % (batch, limit, grid))


def _crop_step(points, pt_off, batch, planes, meta, image_fov):
    """The crop a step runs first: to the camera frustums of ``planes`` [batch,6,4], to the images of ``meta`` with
    ``image_fov``, or none."""
    if planes is not None:
        return ops.frustum_crop(points, pt_off, batch, planes)
    if image_fov:
        return ops.image_fov_crop(points, pt_off, batch, meta)
    return points, pt_off


def _run_step(model, points, pt_off, batch, maxpts, planes=None, meta=None, point_outputs=False, detections=True,
              guided_thr=None, image_fov=False, gt=None):
    """One detector step on the device, no synchronisation; the eager calls and every captured graph build their step
    here.  With ``planes`` [batch,6,4] the frames are full sweeps, cropped to their camera frustums first
    (ops.frustum_crop); with ``image_fov`` they are cropped to their images through ``meta`` (ops.image_fov_crop); then
    forward_device; with ``gt`` (stage_gt's device tensors) the auxiliary network runs too and loss_device puts the
    loss vector [6] in aux["losses"] and its targets in aux["targets"]; with ``meta`` [batch,36] the detections are
    formatted as KITTI rows (ops.kitti_format) into aux["rows"] / aux["n_out"].  Returns forward_device's (det, d_ndet,
    status, aux)."""
    _require_batch(model, batch)
    points, pt_off = _crop_step(points, pt_off, batch, planes, meta, image_fov)
    det, d_ndet, status, aux = model.forward_device(points, pt_off, batch, maxpts,
                                                    point_outputs=point_outputs or gt is not None,
                                                    detections=detections, guided_thr=guided_thr)
    if gt is not None:
        aux["losses"], aux["targets"] = model.loss_device(aux, batch, *gt, None, status)
    if meta is not None:
        aux["rows"], aux["n_out"] = ops.kitti_format(det, d_ndet, meta)
    return det, d_ndet, status, aux


def _stream_through(owner, batches, batch, max_points_per_frame, depth, concurrent, crop, kitti, losses):
    """detect_stream's loop over ``owner``'s slots (a SingleStageDetector's or a DetectorSet's): stage, submit and
    collect round-robin, yielding each batch's results in order."""
    slots, pending = owner._stream_slots, []
    for i, item in enumerate(batches):
        item = tuple(item) if (crop or kitti or losses) else (item,)
        gt = None
        if losses:
            gt, item = owner._gt_inputs(*item[-1], len(item[0])), item[:-1]
        fb = item[0]
        planes = _frame_planes(item[1], len(fb)) if crop else None
        metas = item[-1] if kitti else None
        meta = _meta_blocks(metas, len(fb)) if kitti else None
        counts = [int(p.shape[0]) for p in fb]
        slot = slots[i % depth]
        if len(pending) == depth:                       # the slot we are about to reuse must be drained
            yield owner._collected(*pending.pop(0))
        if not slot.fits(len(fb), counts):
            raise ValueError("batch does not fit the captured shape (batch %d, %d points/frame)" %
                             (batch, max_points_per_frame))
        slot.submit(fb, counts, owner._copy_stream, own_stream=concurrent, planes=planes, meta=meta, gt=gt)
        pending.append((slot, metas))
    for slot, metas in pending:
        yield owner._collected(slot, metas)


def _set_step(dset, points, pt_off, batch, maxpts, planes=None, meta=None, point_outputs=False, image_fov=False,
              gt=None):
    """One DetectorSet step on the device, no synchronisation; the set's eager calls and captured graphs build it here,
    from the parts of _run_step.  Once: the crop, the voxelizer (the members' generators are equal) and the seven
    rulebooks (SpMiddleFHD.sparse_input); per member forward_voxels on the shared voxels and rulebooks; then the
    members' detections gathered per frame (ops.merge_detections) and, with ``meta``, formatted once as KITTI rows.
    The members share the status word.  Returns (det [batch,det_cap,9], d_ndet, status, aux)."""
    assert not point_outputs and gt is None, "a DetectorSet step has no auxiliary outputs or losses"
    lead = dset.models[0]
    _require_batch(lead, batch)
    points, pt_off = _crop_step(points, pt_off, batch, planes, meta, image_fov)
    status = torch.zeros((1,), dtype=torch.int32, device=points.device)
    vox = lead.voxel_generator.generate_device(points, pt_off, batch, maxpts, status)
    _, coors, _, mean, frame_rows = vox
    shared = lead.neck.sparse_input(mean, coors, batch, d_rows=frame_rows[batch:batch + 1], status=status)
    members = [m.forward_voxels(vox, batch, status, sparse_in=shared)[:2] for m in dset.models]
    det, d_ndet = ops.merge_detections(members, dset.label_offsets)
    aux = dict(coors=coors, frame_rows=frame_rows, members=members)
    if meta is not None:
        aux["rows"], aux["n_out"] = ops.kitti_format(det, d_ndet, meta)
    return det, d_ndet, status, aux


def _sweep_step(sweep, points, pt_off, batch, maxpts, planes=None, meta=None, point_outputs=False, image_fov=False,
                gt=None):
    """One CheckpointSweep step on the device, no synchronisation; the sweep's eager calls and captured graphs build it
    here, from the parts of _run_step.  Once: the crop, the voxelizer, the seven rulebooks and the anchor mask, and
    with ``gt`` the nearest voxel centres (member 0's auxiliary network computes them, the others reuse them) and
    loss_targets.  Per member forward_voxels on the shared inputs, loss_device on the shared targets and, with
    ``meta``, the KITTI formatter.  The members share the status word.  Returns (det [K*batch,det_cap,9], d_ndet
    [K*batch], status, aux), the members' blocks one after another, with aux["rows"] / aux["n_out"] likewise and
    aux["losses"] the K loss vectors [K*6]."""
    assert not point_outputs, "a CheckpointSweep step has no auxiliary outputs"
    lead = sweep.models[0]
    _require_batch(lead, batch)
    points, pt_off = _crop_step(points, pt_off, batch, planes, meta, image_fov)
    status = torch.zeros((1,), dtype=torch.int32, device=points.device)
    vox = lead.voxel_generator.generate_device(points, pt_off, batch, maxpts, status)
    _, coors, _, mean, frame_rows = vox
    d_rows = frame_rows[batch:batch + 1]
    mask = lead.anchor_mask(coors, d_rows, batch)
    shared = lead.neck.sparse_input(mean, coors, batch, d_rows=d_rows, status=status)
    dets, ndets, rows, n_out, losses = [], [], [], [], []
    neighbours = targets = None
    for m in sweep.models:
        det, d_ndet, _, aux = m.forward_voxels(vox, batch, status, sparse_in=shared, point_outputs=gt is not None,
                                               mask=mask, neighbours=neighbours)
        dets.append(det)
        ndets.append(d_ndet)
        if gt is not None:
            if targets is None:
                neighbours = aux["idx"], aux["dist2"], aux["points_mean"]
                targets = m.loss_targets(aux, batch, *gt, status)
            losses.append(m.loss_device(aux, batch, *gt, None, status, targets=targets)[0])
        # a member's activations (about 4 GB at batch 16) must be free before the next member allocates its own, so
        # that the step - and its captured graph's private pool - holds one network's, not two
        aux = None
        if meta is not None:
            r, n = ops.kitti_format(det, d_ndet, meta)
            rows.append(r)
            n_out.append(n)
    det, d_ndet = torch.cat(dets), torch.cat(ndets)
    aux = dict(coors=coors, frame_rows=frame_rows)
    if gt is not None:
        aux["losses"] = torch.cat(losses)
    if meta is not None:
        aux["rows"], aux["n_out"] = torch.cat(rows), torch.cat(n_out)
    return det, d_ndet, status, aux


def _pinned_pair(n_points, n_off):
    return (torch.empty((n_points, 4), dtype=torch.float32, pin_memory=True),
            torch.empty((n_off,), dtype=torch.int32, pin_memory=True))


def _stage_into(hp, ho, points_list, counts):
    """Frames -> one pinned buffer + offsets.  Plain numpy memcpy (single thread): torch CPU copies fan out
    over the intra-op thread pool, which costs milliseconds on a many-core host for a 320 KB frame."""
    hp_np, ho_np = hp.numpy(), ho.numpy()
    o = 0
    ho_np[0] = 0
    for i, p in enumerate(points_list):
        n = counts[i]
        if n:
            hp_np[o:o + n] = p[:, :4]
        o += n
        ho_np[i + 1] = o


class _GraphedStep:
    """One captured detector step (_run_step) with static input/output buffers."""

    def __init__(self, model, batch, max_points_per_frame, latency=False, crop=False, kitti=False, point_outputs=False,
                 losses=False, run_step=None):
        """latency=True: this step will run alone on the GPU (enable_cuda_graph / forward_points): the dense convs walk
        the computed tiles first so that the constant-region tiles shorten every layer; False (detect_stream slots,
        several steps in flight): round-robin tiles, the SMs a layer leaves idle serve the other steps.
        crop: the crop kind.  CROP_FRUSTUM (or True): the static points are full sweeps and the graph crops them to the
        frustums given by the static planes [batch,6,4] (ops.frustum_crop) before the step; CROP_IMAGE_FOV (needs
        ``kitti``): the graph crops them to the images of the static meta blocks (ops.image_fov_crop).  The cropped
        frames never exceed the full ones.
        kitti=True: the graph ends with the KITTI result formatter (ops.kitti_format) on the static meta blocks
        [batch,36]; the host copy is its rows and counts instead of the detections.
        point_outputs=True: the step also runs the auxiliary network and copies its outputs and the frame row offsets to
        the host (point_results).
        losses=True: the step also computes the losses of the GT in the static buffers gt [batch,SASSD_GT_CAP_MAX,7],
        its classes, labels and per-frame counts (the true counts: a frame with more boxes raises), and copies the loss
        vector to the host with the detections (loss_results).
        run_step: the step function captured, _run_step's signature (DetectorSet passes _set_step)."""
        dev = next(model.parameters()).device
        self.model, self.batch, self.maxpts = model, int(batch), int(max_points_per_frame)
        self.run_step = _run_step if run_step is None else run_step
        self.cap = self.batch * self.maxpts
        self.crop, self.kitti, self.point_outputs = int(crop), bool(kitti), bool(point_outputs)
        self.losses = bool(losses)
        _crop_kind(self.crop == CROP_FRUSTUM, self.crop == CROP_IMAGE_FOV, self.kitti)
        self.points = torch.zeros((self.cap, 4), dtype=torch.float32, device=dev)
        self.pt_off = torch.zeros((self.batch + 1,), dtype=torch.int32, device=dev)
        self.planes = self.meta = self.gt = None
        if self.crop == CROP_FRUSTUM:
            self.planes = torch.zeros((self.batch, 6, 4), dtype=torch.float64, device=dev)
        if self.kitti:
            self.meta = torch.zeros((self.batch, ops._lib.KITTI_META), dtype=torch.float64, device=dev)
        if self.losses:
            self.h_gt = tuple(torch.from_numpy(a).pin_memory()
                              for a in gt_arrays([np.zeros((0, 7), np.float32)] * self.batch, None, None,
                                                 ops._lib.GT_CAP_MAX))
            self.gt = tuple(h.to(dev) for h in self.h_gt)
        # Scratch buffers private to this graph (the captured kernels bake their addresses in), so that several
        # captured steps can be in flight on different streams without sharing anything but read-only weights.
        self.ws = ops.Workspace()
        self.stream = torch.cuda.Stream(device=dev)
        shared_ws, ops._WS = ops._WS, self.ws
        order0, ops.CONV2D_TILE_ORDER = ops.CONV2D_TILE_ORDER, 1 if latency else 0
        # programmatic dependent launch for the step that runs alone (+2 %); launch attributes are baked into the nodes
        pdl0 = ops._lib.load().sassd_set_pdl(1) if latency else None
        try:
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):   # warm-up: workspaces, weight packs and folded BN get created eagerly
                for _ in range(2):
                    self._step()
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            self.graph = torch.cuda.CUDAGraph()
            self.backgrounds = ops.BACKGROUND_PINS = []       # the captured kernels bake their addresses in
            # A dropped detector lives on in its model <-> captured-step cycles until the cyclic collector runs; a
            # collection during the capture would destroy its CUDA graphs then, which invalidates the capture.  So the
            # dead cycles go now and the collector stays off until the capture ends.
            gc_on = gc.isenabled()
            gc.collect()
            gc.disable()
            try:
                with torch.cuda.graph(self.graph):
                    self.det, self.d_ndet, self.status, self.aux = self._step()
            finally:
                if gc_on:
                    gc.enable()
        finally:
            ops.BACKGROUND_PINS = None
            ops._WS = shared_ws
            ops.CONV2D_TILE_ORDER = order0
            if pdl0 is not None:
                ops._lib.load().sassd_set_pdl(pdl0)
        if self.kitti:
            self.h_rows = torch.empty(self.aux["rows"].shape, dtype=torch.float64, pin_memory=True)
            self.h_nout = torch.empty(self.aux["n_out"].shape, dtype=torch.int32, pin_memory=True)
            self.h_meta = torch.empty(self.meta.shape, dtype=torch.float64, pin_memory=True)
        else:
            self.h_det = torch.empty(self.det.shape, dtype=torch.float32, pin_memory=True)
            self.h_nd = torch.empty(self.d_ndet.shape, dtype=torch.int32, pin_memory=True)
        if self.point_outputs:
            self.h_pts = {k: torch.empty(self.aux[k].shape, dtype=self.aux[k].dtype, pin_memory=True)
                          for k in _POINT_KEYS}
        if self.losses:
            self.h_loss = torch.empty(self.aux["losses"].shape, dtype=torch.float32, pin_memory=True)
        self.h_status = torch.empty((1,), dtype=torch.int32, pin_memory=True)
        self.h_points, self.h_off = _pinned_pair(self.cap, self.batch + 1)
        if self.crop == CROP_FRUSTUM:
            self.h_planes = torch.empty((self.batch, 6, 4), dtype=torch.float64, pin_memory=True)
        self.done = torch.cuda.Event()
        self.loaded = torch.cuda.Event()

    def _step(self):
        return self.run_step(self.model, self.points, self.pt_off, self.batch, self.maxpts, self.planes, self.meta,
                             point_outputs=self.point_outputs, image_fov=self.crop == CROP_IMAGE_FOV, gt=self.gt)

    def fits(self, batch, counts):
        return batch == self.batch and max(counts + [0]) <= self.maxpts

    def load_device(self, points, pt_off):
        """device -> static buffers (for callers whose inputs are already resident)."""
        self.points[: points.shape[0]].copy_(points, non_blocking=True)
        self.pt_off.copy_(pt_off, non_blocking=True)

    def replay(self):
        self.graph.replay()
        return self.det, self.d_ndet, self.status

    def run_host(self, hp, ho, total, planes=None, meta=None, gt=None):
        """pinned host points in, numpy detections (or KITTI rows) out: H2D, one graph launch, D2H, one stream sync."""
        self._upload(hp, ho, total, planes, meta, gt)
        self.graph.replay()
        self._download()
        torch.cuda.current_stream().synchronize()
        return self.unpack()

    def _upload(self, hp, ho, total, planes, meta, gt=None):
        """H2D of a step's inputs into the static buffers on the current stream: ``total`` points of the pinned ``hp``,
        the pinned offsets ``ho`` and, for a crop / formatting / loss step, the numpy planes / meta blocks / gt_arrays'
        inputs."""
        self.points[:total].copy_(hp[:total], non_blocking=True)
        self.pt_off.copy_(ho, non_blocking=True)
        if self.crop == CROP_FRUSTUM:
            self.h_planes.numpy()[...] = planes
            self.planes.copy_(self.h_planes, non_blocking=True)
        if self.kitti:
            self.h_meta.numpy()[...] = meta
            self.meta.copy_(self.h_meta, non_blocking=True)
        if self.losses:
            for h, d, a in zip(self.h_gt, self.gt, gt_arrays(*gt, gt_cap=ops._lib.GT_CAP_MAX)):
                h.numpy()[...] = a
                d.copy_(h, non_blocking=True)

    def _download(self):
        """D2H of the step's result on the current stream: the KITTI rows and counts of a formatting step, else the
        detections and counts; the loss vector of a loss step; and the status word."""
        if self.kitti:
            self.h_rows.copy_(self.aux["rows"], non_blocking=True)
            self.h_nout.copy_(self.aux["n_out"], non_blocking=True)
        else:
            self.h_det.copy_(self.det, non_blocking=True)
            self.h_nd.copy_(self.d_ndet, non_blocking=True)
        if self.point_outputs:
            for k, h in self.h_pts.items():
                h.copy_(self.aux[k], non_blocking=True)
        if self.losses:
            self.h_loss.copy_(self.aux["losses"], non_blocking=True)
        self.h_status.copy_(self.status, non_blocking=True)

    # ---- asynchronous use (SingleStageDetector.detect_stream): submit() ... collect()
    def submit(self, points_list, counts, copy_stream, own_stream=False, planes=None, meta=None, gt=None):
        """Stage into this slot's pinned buffer, H2D on the copy stream, then replay + D2H on the current stream or,
        with ``own_stream``, on this slot's stream so that consecutive steps overlap on the GPU."""
        _stage_into(self.h_points, self.h_off, points_list, counts)
        cur = self.stream if own_stream else torch.cuda.current_stream()
        with torch.cuda.stream(copy_stream):
            self._upload(self.h_points, self.h_off, sum(counts), planes, meta, gt)
            self.loaded.record(copy_stream)
        cur.wait_event(self.loaded)
        with torch.cuda.stream(cur):
            self.graph.replay()
            self._download()
            self.done.record(cur)

    def collect(self):
        self.done.synchronize()
        return self.unpack()

    def point_results(self):
        """The last run's aux outputs, per frame (forward_points(point_outputs=True))."""
        return _split_points(*(self.h_pts[k].numpy() for k in _POINT_KEYS))

    def loss_results(self):
        """The last run's losses (forward_points with GT, detect_stream(losses=True)); read after unpack, which checks
        the status word."""
        return _loss_dict(self.h_loss)

    def unpack(self):
        ops._lib.raise_on_status(self.h_status.numpy()[0])
        if self.kitti:      # (rows, n_out): results.annos_from_rows
            return self.h_rows.numpy().copy(), self.h_nout.numpy().copy()
        return split_detections(self.h_det.numpy(), self.h_nd.numpy())

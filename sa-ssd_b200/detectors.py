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
    device first (the reference crops them offline into ``velodyne_reduced``).  With ``metas``
    the step also formats its detections as KITTI annotations on the device (ops.kitti_format).
"""
import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from . import builder, ops
from .results import annos_from_rows, meta_block
from .single_stage_heads import unpack_detections


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
        self._graph = None
        self._crop_graph = None
        self._kitti_graphs = {}           # crop -> captured step that also formats KITTI rows (forward_points metas=)
        self._graph_args = None
        self._stream_slots = None
        self._stream_key = None
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
        self._drop_captured_graphs()

    def _drop_captured_graphs(self):
        """Captured steps bake in the device addresses of packed weights, folded BN vectors and layer constants and
        the kernel selection; anything that changes those must force a re-capture."""
        self._graph = None
        self._crop_graph = None
        self._kitti_graphs = {}
        self._stream_slots = None
        self._stream_key = None

    def refresh_packed_weights(self):
        """Called after parameters were (re)loaded (checkpoint.load_state_dict_into).  Packed / folded tensors are
        version-checked on eager use, but a CUDA-graph replay never re-checks: drop every captured step (the
        single-step graph of enable_cuda_graph and the detect_stream slots) so the next call re-captures with the
        new weights."""
        self._drop_captured_graphs()

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
            raise NotImplementedError("training (forward_train, single_stage.py:75-108) is out of scope")
        return self.forward_test(img, img_meta, **kwargs)

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

    def forward_device(self, points, pt_off, batch, max_points_per_frame):
        """Everything on the device, no synchronisation.  points [Ncap,4], pt_off [batch+1] int32.
        Returns (det [B,det_cap,9], d_ndet [B], status [1], aux dict)."""
        dev = points.device
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        vg, aset = self.voxel_generator, self.anchor_set
        voxels, coors, num, mean, frame_rows = vg.generate_device(points, pt_off, batch, max_points_per_frame, status)
        d_rows = frame_rows[batch:batch + 1]
        # anchors_mask only feeds the guided-anchor selection: run it on a side stream, next to the backbone
        main = torch.cuda.current_stream()
        if self._mask_stream is None:
            self._mask_stream = torch.cuda.Stream(device=dev)
        self._mask_stream.wait_stream(main)
        with torch.cuda.stream(self._mask_stream):
            mask = aset.mask_device(coors, d_rows, batch)
        y, conv6, xs = self.neck.forward_nhwc(mean, coors, batch, d_rows=d_rows, status=status)
        main.wait_stream(self._mask_stream)
        head = self.rpn_head.forward_nhwc(y)
        anchors, _ = aset.device_tensors()
        boxes, labels, index, d_k = self.rpn_head.guided_anchors_device(head, anchors, mask, self.guided_thr, status)
        scores = self.extra_head.forward_device(conv6, boxes, d_k)
        det, d_ndet = self.extra_head.rescore_device(boxes, scores, labels, d_k, self.test_cfg.extra, status)
        aux = dict(voxels=voxels, coors=coors, num_points=num, mean=mean, frame_rows=frame_rows, mask=mask, x=y,
                   conv6=conv6, head=head, guided=boxes, guided_labels=labels, guided_index=index, d_k=d_k,
                   ps_scores=scores, sparse=xs)
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
        launch.  Steps whose shape does not fit fall back to the eager path.  Calls with ``frustum_planes`` replay a
        second graph, captured on their first use, that runs the crop and the step; there ``max_points_per_frame`` bounds
        the full sweeps (e.g. 131072).  Calls with ``metas`` replay a graph, again captured on first use, that ends with
        the KITTI result formatter."""
        self._graph_args = (int(batch), int(max_points_per_frame))
        self._graph = _GraphedStep(self, batch, max_points_per_frame, latency=True)
        return self._graph

    def disable_cuda_graph(self):
        self._graph = None
        self._crop_graph = None
        self._kitti_graphs = {}
        self._graph_args = None

    def detect_stream(self, batches, batch, max_points_per_frame=32768, depth=4, concurrent=True, crop=False,
                      kitti=False):
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
        result formatter and each yield is the batch's annotation dicts (kitti_bbox2results' format)."""
        ops.require_cuda()
        if kitti and self.class_names is None:
            raise ValueError("detect_stream(kitti=True) needs class_names")
        key = (batch, max_points_per_frame, depth, bool(crop), bool(kitti))
        if self._stream_key != key or self._stream_slots is None:
            self._stream_slots = [_GraphedStep(self, batch, max_points_per_frame, crop=crop, kitti=kitti)
                                  for _ in range(depth)]
            self._copy_stream = torch.cuda.Stream()
            self._stream_key = key
        slots, pending = self._stream_slots, []
        for i, item in enumerate(batches):
            item = tuple(item) if (crop or kitti) else (item,)
            fb = item[0]
            planes = _frame_planes(item[1], len(fb)) if crop else None
            metas = item[-1] if kitti else None
            meta = _meta_blocks(metas, len(fb)) if kitti else None
            counts = [int(p.shape[0]) for p in fb]
            slot = slots[i % depth]
            if len(pending) == depth:                       # the slot we are about to reuse must be drained
                yield self._collected(*pending.pop(0))
            if not slot.fits(len(fb), counts):
                raise ValueError("batch does not fit the captured shape (batch %d, %d points/frame)" %
                                 (batch, max_points_per_frame))
            slot.submit(fb, counts, self._copy_stream, own_stream=concurrent, planes=planes, meta=meta)
            pending.append((slot, metas))
        for slot, metas in pending:
            yield self._collected(slot, metas)

    def _collected(self, slot, metas):
        """Wait for a slot's step and convert its host copy into the caller's per-frame results."""
        out = slot.collect()
        if slot.kitti:
            return annos_from_rows(*out, self.class_names, [m["sample_idx"] for m in metas])
        return [dict(boxes_lidar=b, scores=s, label_preds=l) for b, s, l in zip(*out)]

    def forward_points(self, points_list, return_aux=False, frustum_planes=None, metas=None):
        """Raw points in (list of [N_i,>=4] numpy arrays), detections out: per frame a dict of
        boxes_lidar [D,7], scores [D], label_preds [D] (or None entries when nothing survives).
        ``frustum_planes``: one float64 [6,4] array per frame (frustum.camera_frustum_planes).  The frames are then
        full sweeps; each is cropped to its camera frustum on the device, in point order (ops.frustum_crop), and the
        step runs on what is left, as on the reference's offline-cropped ``velodyne_reduced`` clouds.
        ``metas``: one ``img_meta``-style dict per frame ('calib' a results.Calibration, 'img_shape', 'sample_idx').
        The detections are then formatted on the device (ops.kitti_format) and the call returns, like forward_test,
        one KITTI annotation dict per frame; ``class_names`` must be set.  With ``return_aux`` the aux dict also holds
        the unformatted detections (det, ndet)."""
        ops.require_cuda()
        if self.voxel_generator is None or self.anchor_set is None:
            raise RuntimeError("call attach_data_pipeline(voxel_generator, anchor_set) first")
        if metas is not None and self.class_names is None:
            raise ValueError("forward_points(metas=) needs class_names")
        dev = next(self.parameters()).device
        planes = None if frustum_planes is None else _frame_planes(frustum_planes, len(points_list))
        meta = None if metas is None else _meta_blocks(metas, len(points_list))
        hp, ho, counts = self.stage_points(points_list)
        if meta is not None:
            crop = planes is not None
            if crop not in self._kitti_graphs and self._graph_args is not None:
                self._kitti_graphs[crop] = _GraphedStep(self, *self._graph_args, latency=True, crop=crop, kitti=True)
            g = self._kitti_graphs.get(crop)
        elif planes is None:
            if self._graph is None and self._graph_args is not None:     # dropped by a weight / precision change
                self._graph = _GraphedStep(self, *self._graph_args, latency=True)
            g = self._graph
        else:
            if self._crop_graph is None and self._graph_args is not None:
                self._crop_graph = _GraphedStep(self, *self._graph_args, latency=True, crop=True)
            g = self._crop_graph
        if g is not None and not return_aux and g.fits(len(points_list), counts):
            out = g.run_host(hp, ho, sum(counts), planes, meta)
            if meta is not None:
                return annos_from_rows(*out, self.class_names, [m["sample_idx"] for m in metas])
            return [dict(boxes_lidar=b, scores=s, label_preds=l) for b, s, l in zip(*out)]
        points = hp.to(dev, non_blocking=True)
        pt_off = ho.to(dev, non_blocking=True)
        if planes is not None:
            points, pt_off = ops.frustum_crop(points, pt_off, len(points_list), torch.from_numpy(planes).to(dev))
        det, d_ndet, status, aux = self.forward_device(points, pt_off, len(points_list), max(counts + [1]))
        if meta is not None:
            rows, n_out = ops.kitti_format(det, d_ndet, torch.from_numpy(meta).to(dev))
            word = int(status.item())
            if word:
                raise ops._lib.SassdError("capacity overflow on device: %s" % ops._lib.decode_flags(word))
            out = annos_from_rows(rows.cpu().numpy(), n_out.cpu().numpy(), self.class_names,
                                  [m["sample_idx"] for m in metas])
            aux.update(det=det, ndet=d_ndet)
            return (out, aux) if return_aux else out
        bbs, scs, lbs = unpack_detections(det, d_ndet, status)
        out = [dict(boxes_lidar=b, scores=s, label_preds=l) for b, s, l in zip(bbs, scs, lbs)]
        return (out, aux) if return_aux else out


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
    """One captured step of SingleStageDetector.forward_device with static input/output buffers."""

    def __init__(self, model, batch, max_points_per_frame, latency=False, crop=False, kitti=False):
        """latency=True: this step will run alone on the GPU (enable_cuda_graph / forward_points): the dense convs walk
        the computed tiles first so that the constant-region tiles shorten every layer; False (detect_stream slots,
        several steps in flight): round-robin tiles, the SMs a layer leaves idle serve the other steps.
        crop=True: the static points are full sweeps and the graph crops them to the frustums given by the static
        planes [batch,6,4] (ops.frustum_crop) before the step; the cropped frames never exceed the full ones.
        kitti=True: the graph ends with the KITTI result formatter (ops.kitti_format) on the static meta blocks
        [batch,36]; the host copy is its rows and counts instead of the detections."""
        dev = next(model.parameters()).device
        self.model, self.batch, self.maxpts = model, int(batch), int(max_points_per_frame)
        self.cap = self.batch * self.maxpts
        self.crop, self.kitti = bool(crop), bool(kitti)
        self.points = torch.zeros((self.cap, 4), dtype=torch.float32, device=dev)
        self.pt_off = torch.zeros((self.batch + 1,), dtype=torch.int32, device=dev)
        if self.crop:
            self.planes = torch.zeros((self.batch, 6, 4), dtype=torch.float64, device=dev)
        if self.kitti:
            self.meta = torch.zeros((self.batch, ops._lib.KITTI_META), dtype=torch.float64, device=dev)
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
            with torch.cuda.graph(self.graph):
                self.det, self.d_ndet, self.status, self.aux = self._step()
        finally:
            ops.BACKGROUND_PINS = None
            ops._WS = shared_ws
            ops.CONV2D_TILE_ORDER = order0
            if pdl0 is not None:
                ops._lib.load().sassd_set_pdl(pdl0)
        if self.kitti:
            self.h_rows = torch.empty(self.rows.shape, dtype=torch.float64, pin_memory=True)
            self.h_nout = torch.empty(self.n_out.shape, dtype=torch.int32, pin_memory=True)
            self.h_meta = torch.empty(self.meta.shape, dtype=torch.float64, pin_memory=True)
        else:
            self.h_det = torch.empty(self.det.shape, dtype=torch.float32, pin_memory=True)
            self.h_nd = torch.empty(self.d_ndet.shape, dtype=torch.int32, pin_memory=True)
        self.h_status = torch.empty((1,), dtype=torch.int32, pin_memory=True)
        self.h_points, self.h_off = _pinned_pair(self.cap, self.batch + 1)
        if self.crop:
            self.h_planes = torch.empty((self.batch, 6, 4), dtype=torch.float64, pin_memory=True)
        self.done = torch.cuda.Event()
        self.loaded = torch.cuda.Event()

    def _step(self):
        points, pt_off = self.points, self.pt_off
        if self.crop:
            points, pt_off = ops.frustum_crop(points, pt_off, self.batch, self.planes)
        det, d_ndet, status, aux = self.model.forward_device(points, pt_off, self.batch, self.maxpts)
        if self.kitti:
            self.rows, self.n_out = ops.kitti_format(det, d_ndet, self.meta)
        return det, d_ndet, status, aux

    def fits(self, batch, counts):
        return batch == self.batch and max(counts + [0]) <= self.maxpts

    def load_device(self, points, pt_off):
        """device -> static buffers (for callers whose inputs are already resident)."""
        self.points[: points.shape[0]].copy_(points, non_blocking=True)
        self.pt_off.copy_(pt_off, non_blocking=True)

    def replay(self):
        self.graph.replay()
        return self.det, self.d_ndet, self.status

    def run_host(self, hp, ho, total, planes=None, meta=None):
        """pinned host points in, numpy detections (or KITTI rows) out: H2D, one graph launch, D2H, one stream sync."""
        self.points[:total].copy_(hp[:total], non_blocking=True)
        self.pt_off.copy_(ho, non_blocking=True)
        if self.crop:
            self.h_planes.numpy()[...] = planes
            self.planes.copy_(self.h_planes, non_blocking=True)
        if self.kitti:
            self.h_meta.numpy()[...] = meta
            self.meta.copy_(self.h_meta, non_blocking=True)
        self.graph.replay()
        self._download()
        torch.cuda.current_stream().synchronize()
        return self.unpack()

    def _download(self):
        """D2H of the step's result on the current stream: the KITTI rows and counts of a formatting step, else the
        detections and counts; and the status word."""
        if self.kitti:
            self.h_rows.copy_(self.rows, non_blocking=True)
            self.h_nout.copy_(self.n_out, non_blocking=True)
        else:
            self.h_det.copy_(self.det, non_blocking=True)
            self.h_nd.copy_(self.d_ndet, non_blocking=True)
        self.h_status.copy_(self.status, non_blocking=True)

    # ---- asynchronous use (SingleStageDetector.detect_stream): submit() ... collect()
    def submit(self, points_list, counts, copy_stream, own_stream=False, planes=None, meta=None):
        """Stage into this slot's pinned buffer, H2D on the copy stream, then replay + D2H on the current stream or,
        with ``own_stream``, on this slot's stream so that consecutive steps overlap on the GPU."""
        _stage_into(self.h_points, self.h_off, points_list, counts)
        if self.crop:
            self.h_planes.numpy()[...] = planes
        if self.kitti:
            self.h_meta.numpy()[...] = meta
        total = sum(counts)
        cur = self.stream if own_stream else torch.cuda.current_stream()
        with torch.cuda.stream(copy_stream):
            self.points[:total].copy_(self.h_points[:total], non_blocking=True)
            self.pt_off.copy_(self.h_off, non_blocking=True)
            if self.crop:
                self.planes.copy_(self.h_planes, non_blocking=True)
            if self.kitti:
                self.meta.copy_(self.h_meta, non_blocking=True)
            self.loaded.record(copy_stream)
        cur.wait_event(self.loaded)
        with torch.cuda.stream(cur):
            self.graph.replay()
            self._download()
            self.done.record(cur)

    def collect(self):
        self.done.synchronize()
        return self.unpack()

    def unpack(self):
        word = int(self.h_status.numpy()[0])
        if word:
            raise ops._lib.SassdError("capacity overflow on device: %s" % ops._lib.decode_flags(word))
        if self.kitti:      # (rows, n_out): results.annos_from_rows
            return self.h_rows.numpy().copy(), self.h_nout.numpy().copy()
        det, n = self.h_det.numpy(), self.h_nd.numpy()
        bbs, scs, lbs = [], [], []
        for b in range(det.shape[0]):
            k = int(n[b])
            if k == 0:
                bbs.append(None); scs.append(None); lbs.append(None)
                continue
            bbs.append(det[b, :k, :7].copy()); scs.append(det[b, :k, 7].copy())
            lbs.append(det[b, :k, 8].astype(np.int64))
        return bbs, scs, lbs

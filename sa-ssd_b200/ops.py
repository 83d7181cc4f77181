"""Functional wrappers over the C ABI (include/sassd_b200.h) on torch CUDA tensors.

torch is plumbing here (device memory, streams); every computation is a
hand-written sm_90a kernel in csrc/.  All wrappers are asynchronous on the
current torch stream and keep data-dependent sizes on the device (``d_rows``
style int32 tensors) — nothing in this module synchronises.
"""
import collections
import ctypes
import os
import math

import numpy as np
import torch

from . import lib as _lib
from .lib import Conv2dDesc, SpconvDesc  # noqa: E402
from .lib import (GCONV_CONV2D, GCONV_ROWS, GCONV_TABLE, PREC_F16X3, PREC_FP32, PREC_TF32X3, GConvDesc, VoxelParams,
                  check)

NMS_CAP = 4096
# Product default: every conv on the tensor-core (wgmma) kernels with the fp32-accurate 3xFP16 operand split (csrc/spconv_split.cu,
# csrc/conv2d_tma.cu).  PREC_FP32 (CUDA-core FFMA) and PREC_TF32X3 stay selectable per model
# (SingleStageDetector.set_precision) for bisecting.
DEFAULT_PRECISION = PREC_F16X3


def _L():
    return _lib.load()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    if t is None:
        return ctypes.c_void_p(0)
    assert t.is_cuda and t.is_contiguous(), "sassd ops need contiguous CUDA tensors"
    return ctypes.c_void_p(t.data_ptr())


def require_cuda():
    if not torch.cuda.is_available():
        raise _lib.SassdError("sassd_b200 needs a CUDA device (sm_90a); there is no CPU fallback")


def next_pow2(n):
    return 1 << max(1, int(math.ceil(math.log2(max(2, n)))))


# --- launch accounting / optional per-call CUDA-event timing (bench.py) ---------------
# kernels launched by each C-ABI entry point (memsets not counted)
_KERNELS = {"sassd_voxelize": 4, "sassd_voxel_mean": 1, "sassd_frustum_crop": 1, "sassd_image_fov_crop": 1, "sassd_points_in_rbboxes": 1, "sassd_augment_drop_points": 1, "sassd_augment_noise_search": 1, "sassd_augment_assemble": 1, "sassd_anchor_mask": 4, "sassd_hash_build": 1,
            "sassd_rulebook_subm": 1, "sassd_rulebook_conv_outputs": 2, "sassd_rulebook_conv_outputs_hash": 2, "sassd_rulebook_conv_nbr": 1,
            "sassd_rulebook_pairs": 1, "sassd_gconv": 1, "sassd_gconv_pack": 1, "sassd_spconv_pack": 1, "sassd_rotate_overlap_eval": 1, "sassd_kitti_eval_flags": 1, "sassd_kitti_eval_flags_ranged": 1, "sassd_kitti_eval_assign": 1, "sassd_kitti_eval_overlaps": 1, "sassd_kitti_eval_match": 3, "sassd_kitti_scan_labels": 1, "sassd_kitti_parse_labels": 2, "sassd_conv2d_pack": 1, "sassd_conv2d_f16x3": 1, "sassd_conv2d_f16x3_occ": 1, "sassd_conv2d_f16x3_occ_bg": 1, "sassd_conv2d_f16x3_occ_bg_status": 1, "sassd_gconv_status": 1, "sassd_spconv_f16x3_status": 1, "sassd_features_to_split_status": 1, "sassd_sparse_to_bev_split_status": 1, "sassd_spconv_f16x3": 1, "sassd_features_to_split": 1, "sassd_split_rows_to_bev": 1, "sassd_sparse_to_bev_split": 1, "sassd_sparse_to_bev": 1, "sassd_decode_select": 2,
            "sassd_pswarp": 1, "sassd_rescore_nms": 3, "sassd_kitti_format": 1, "sassd_merge_detections": 1, "sassd_three_nn": 1, "sassd_point_aux_head": 1, "sassd_nms_mask": 1, "sassd_nms_sorted": 2,
            "sassd_boxes_iou_bev": 1, "sassd_points_in_boxes": 2, "sassd_assign_rpn": 3, "sassd_assign_pswarp": 3,
            "sassd_rpn_loss": 2, "sassd_pswarp_loss": 2, "sassd_aux_loss": 2}
LAUNCHES = 0          # running count of kernels launched through this module
PROFILE = None        # set to a list to collect (name, label, start_event, end_event)


def _call(name, label, *args):
    global LAUNCHES
    LAUNCHES += _KERNELS[name]
    fn = getattr(_L(), name)
    if PROFILE is None:
        check(fn(*args), name)
        return
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    check(fn(*args), name)
    e1.record()
    PROFILE.append((name, label, e0, e1))


class Workspace:
    """Grow-only byte buffers keyed by purpose (the C ABI never allocates)."""

    def __init__(self):
        self._bufs = {}

    def get(self, key, nbytes, device, zeroed=False):
        """zeroed: a new buffer starts zero-filled (for kernels that keep counters in it and leave them zero)."""
        buf = self._bufs.get(key)
        if buf is None or buf.numel() < nbytes or buf.device != device:
            buf = (torch.zeros if zeroed else torch.empty)(max(int(nbytes), 256), dtype=torch.uint8, device=device)
            self._bufs[key] = buf
        return buf


_WS = Workspace()


# ---------------------------------------------------------------------------- voxelize
def make_voxel_params(voxel_size, pc_range, max_points, max_voxels):
    vs = np.asarray(voxel_size, np.float32)
    rg = np.asarray(pc_range, np.float32)
    grid = np.round((rg[3:] - rg[:3]) / vs).astype(np.int64)   # voxel_generator.py:13-15
    p = VoxelParams()
    for j in range(3):
        p.voxel_size[j] = float(vs[j]); p.range_min[j] = float(rg[j]); p.grid[j] = int(grid[j])
    p.max_points = int(max_points); p.max_voxels = int(max_voxels)
    return p, grid


def voxelize(points, pt_off, batch, params, rows_cap, slots_per_frame, status, want_mean=True, ws=None):
    """points [Ncap,4] f32, pt_off [batch+1] i32 (device).  Returns capacity-sized
    (voxels, coors, num_points, mean, frame_rows[batch+1])."""
    dev = points.device
    n_cap = points.shape[0]
    voxels = torch.empty((rows_cap, params.max_points, 4), dtype=torch.float32, device=dev)
    coors = torch.empty((rows_cap, 4), dtype=torch.int32, device=dev)
    num = torch.empty((rows_cap,), dtype=torch.int32, device=dev)
    mean = torch.empty((rows_cap, 4), dtype=torch.float32, device=dev) if want_mean else None
    frame_rows = torch.empty((batch + 1,), dtype=torch.int32, device=dev)
    nbytes = _L().sassd_voxelize_workspace_bytes(n_cap, batch, slots_per_frame)
    w = (ws or _WS).get("voxelize", nbytes, dev)
    _call("sassd_voxelize", None, _ptr(points), _ptr(pt_off), n_cap, batch, ctypes.byref(params), slots_per_frame,
                              _ptr(voxels), _ptr(coors), _ptr(num), _ptr(mean), rows_cap, _ptr(frame_rows),
                              _ptr(status), _ptr(w), w.numel(), _stream())
    return voxels, coors, num, mean, frame_rows


def frustum_crop(points, pt_off, batch, planes, ws=None):
    """points [Ncap,4] f32, pt_off [batch+1] i32, planes [batch,6,4] f64 (device; frustum.camera_frustum_planes).
    Returns (points_out [Ncap,4], pt_off_out [batch+1]): each frame's points inside its camera frustum, in input
    order, frames concatenated.  Rows past pt_off_out[batch] are left unwritten."""
    dev = points.device
    n_cap = points.shape[0]
    assert planes.dtype == torch.float64 and tuple(planes.shape) == (batch, 6, 4), "planes must be float64 [batch,6,4]"
    out = torch.empty_like(points)
    off = torch.empty((batch + 1,), dtype=torch.int32, device=dev)
    nbytes = _L().sassd_frustum_crop_workspace_bytes(n_cap, batch)
    w = (ws or _WS).get("frustum", nbytes, dev)
    _call("sassd_frustum_crop", None, _ptr(points), _ptr(pt_off), n_cap, batch, _ptr(planes), _ptr(out), _ptr(off),
          _ptr(w), w.numel(), _stream())
    return out, off


IMAGE_FOV_CLIP_X = 0.1      # the reference's clip distance for raw drives (mmdet/datasets/kitti.py:394)


def image_fov_crop(points, pt_off, batch, meta, clip_x=IMAGE_FOV_CLIP_X, ws=None):
    """points [Ncap,4] f32, pt_off [batch+1] i32, meta [batch,36] f64 (device; results.meta_block).  Returns
    (points_out [Ncap,4], pt_off_out [batch+1]): each frame's points that project into its image (0 <= u < img_w,
    0 <= v < img_h) and lie in front of x = clip_x (compared in fp32), in input order, frames concatenated; the
    reference's get_lidar_in_image_fov.  Rows past pt_off_out[batch] are left unwritten."""
    dev = points.device
    n_cap = points.shape[0]
    assert meta.dtype == torch.float64 and tuple(meta.shape) == (batch, _lib.KITTI_META), \
        "meta must be float64 [batch,%d]" % _lib.KITTI_META
    out = torch.empty_like(points)
    off = torch.empty((batch + 1,), dtype=torch.int32, device=dev)
    nbytes = _L().sassd_frustum_crop_workspace_bytes(n_cap, batch)
    w = (ws or _WS).get("frustum", nbytes, dev)      # the same look-back descriptors as the frustum crop
    _call("sassd_image_fov_crop", None, _ptr(points), _ptr(pt_off), n_cap, batch, _ptr(meta), float(clip_x), _ptr(out),
          _ptr(off), _ptr(w), w.numel(), _stream())
    return out, off


def points_in_rbboxes(points, pt_off, batch, planes, centres, nbox, gather_cap, status=None, ws=None):
    """points [Ncap,4] f32, pt_off [batch+1] i32 (device; frustum_crop's outputs), planes [batch,box_cap,6,4] f64,
    centres [batch,box_cap,3] f64, nbox [batch] i32 (device; create_data.box_planes).  Returns (counts
    [batch,box_cap] i32, seg_off [batch*box_cap+1] i32, gathered [gather_cap,4] f32, status [1] i32): the members of
    box (b, j) are gathered[seg_off[b*box_cap+j]:][:counts[b,j]] in input order, x, y, z relative to the box centre
    (the reference's points_in_rbbox and gt database rows).  Raise on ``status`` (lib.raise_on_status) after the
    caller's sync: GATHER_CAP when more than gather_cap rows were due, GT_CAP when nbox exceeds box_cap."""
    dev = points.device
    n_cap = points.shape[0]
    box_cap = planes.shape[1] if planes.dim() == 4 else -1
    assert planes.dtype == torch.float64 and tuple(planes.shape) == (batch, box_cap, 6, 4), \
        "planes must be float64 [batch,box_cap,6,4]"
    assert centres.dtype == torch.float64 and tuple(centres.shape) == (batch, box_cap, 3), \
        "centres must be float64 [batch,box_cap,3]"
    assert nbox.dtype == torch.int32 and tuple(nbox.shape) == (batch,), "nbox must be int32 [batch]"
    if status is None:
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
    counts = torch.empty((batch, box_cap), dtype=torch.int32, device=dev)
    seg_off = torch.empty((batch * box_cap + 1,), dtype=torch.int32, device=dev)
    gathered = torch.empty((max(int(gather_cap), 1), 4), dtype=torch.float32, device=dev)
    nbytes = _L().sassd_points_in_rbboxes_workspace_bytes(n_cap, batch, box_cap)
    w = (ws or _WS).get("rbboxes", nbytes, dev)
    _call("sassd_points_in_rbboxes", None, _ptr(points), _ptr(pt_off), n_cap, batch, _ptr(planes), _ptr(centres),
          _ptr(nbox), box_cap, _ptr(counts), _ptr(seg_off), _ptr(gathered), int(gather_cap), _ptr(status), _ptr(w),
          w.numel(), _stream())
    return counts, seg_off, gathered, status


def augment_drop_points(points, pt_off, batch, planes, box_off, ws=None):
    """points [Ncap,4] f32, pt_off [batch+1] i32, planes [boxes,6,4] f32, box_off [batch+1] i32 (device).  Returns
    (points_out [Ncap,4], pt_off_out [batch+1]): each frame's points outside every one of its boxes under the fp32
    plane test, in input order (the scene crop of the reference's prepare_train_img)."""
    dev = points.device
    n_cap = points.shape[0]
    assert planes.dtype == torch.float32 and planes.shape[1:] == (6, 4), "planes must be float32 [boxes,6,4]"
    out = torch.empty_like(points)
    off = torch.empty((batch + 1,), dtype=torch.int32, device=dev)
    nbytes = _L().sassd_frustum_crop_workspace_bytes(n_cap, batch)
    w = (ws or _WS).get("frustum", nbytes, dev)
    _call("sassd_augment_drop_points", None, _ptr(points), _ptr(pt_off), n_cap, batch, _ptr(planes), _ptr(box_off),
          _ptr(out), _ptr(off), _ptr(w), w.numel(), _stream())
    return out, off


def augment_noise_search(boxes, box_trig, box_off, batch, try_trig, loc, status):
    """boxes [K,5] f32 (x, y, w, l, ry), box_trig [K,2] f32, box_off [batch+1] i32, try_trig [K,T,2] f32, loc [K,T,3]
    f64 (device).  Returns sel [K] i32: each box's first collision-free try, or -1 (the reference's noise_per_box)."""
    tries = loc.shape[1]
    sel = torch.empty((boxes.shape[0],), dtype=torch.int32, device=boxes.device)
    _call("sassd_augment_noise_search", None, _ptr(boxes), _ptr(box_trig), _ptr(box_off), batch, tries, _ptr(try_trig),
          _ptr(loc), _ptr(sel), _ptr(status), _stream())
    return sel


def augment_assemble(kept, kept_off, batch, srow_off, srec_off, srec_db, srec_ctr, db, box_off, planes, centres, sel,
                     try_trig, loc, frame_tf, out_cap, status, dz=None):
    """The augmented cloud of every frame: its sampled database rows, then the kept scene rows, each moved by its box's
    noise and the frame's flip, rotation and scaling (csrc/augment.cu).  ``dz`` [records] f64 (optional): each sampled
    record's height move onto its frame's road plane, subtracted from its rows' z after the centre add.  Returns
    (points [out_cap,4], pt_off [batch+1]); POINTS_CAP in ``status`` when the rows exceed out_cap."""
    if dz is not None:
        assert dz.dtype == torch.float64 and dz.numel() >= srec_db.numel(), "dz must be float64 [records]"
    dev = kept.device
    out = torch.empty((max(int(out_cap), 1), 4), dtype=torch.float32, device=dev)
    off = torch.empty((batch + 1,), dtype=torch.int32, device=dev)
    _call("sassd_augment_assemble", None, _ptr(kept), _ptr(kept_off), batch, _ptr(srow_off), _ptr(srec_off),
          srec_db.numel(), _ptr(srec_db), _ptr(srec_ctr), _ptr(dz), _ptr(db), _ptr(box_off), _ptr(planes), _ptr(centres),
          _ptr(sel), loc.shape[1], _ptr(try_trig), _ptr(loc), _ptr(frame_tf), int(out_cap), _ptr(out), _ptr(off),
          _ptr(status), _stream())
    return out, off


def voxel_mean(voxels, num_points, d_rows=None):
    rows, maxp = voxels.shape[0], voxels.shape[1]
    mean = torch.empty((rows, 4), dtype=torch.float32, device=voxels.device)
    _call("sassd_voxel_mean", None, _ptr(voxels), _ptr(num_points), _ptr(d_rows), rows, maxp, _ptr(mean), _stream())
    return mean


def anchor_mask(coors, d_rows, batch, H, W, rects, threshold=1, ws=None):
    dev = coors.device
    na = rects.shape[0]
    mask = torch.empty((batch, na), dtype=torch.uint8, device=dev)
    nbytes = _L().sassd_anchor_mask_workspace_bytes(batch, H, W)
    w = (ws or _WS).get("amask", nbytes, dev)
    _call("sassd_anchor_mask", None, _ptr(coors), _ptr(d_rows), coors.shape[0], batch, H, W, _ptr(rects), na,
                                 int(threshold), _ptr(mask), _ptr(w), w.numel(), _stream())
    return mask


# ---------------------------------------------------------------------------- rulebooks
class HashIndex:
    def __init__(self, rows_cap, device):
        self.slots = next_pow2(2 * max(rows_cap, 1))
        self.keys = torch.empty((self.slots,), dtype=torch.int32, device=device)
        self.vals = torch.empty((self.slots,), dtype=torch.int32, device=device)


def hash_build(index, coors, d_rows, batch, shape, status):
    D, H, W = shape
    _call("sassd_hash_build", None, _ptr(coors), _ptr(d_rows), coors.shape[0], batch, D, H, W, _ptr(index.keys),
                                _ptr(index.vals), index.slots, _ptr(status), _stream())
    return index


def _tile_mask_buffer(rows_cap, device):
    """int32 per 128-row tile: which of the 27 taps occur in the tile (written by the rulebook kernels, read by
    spconv_split to skip absent taps)."""
    n = (rows_cap + _lib.SPCONV_TILE_ROWS - 1) // _lib.SPCONV_TILE_ROWS
    return torch.empty((max(n, 1),), dtype=torch.int32, device=device)


def rulebook_subm(coors, d_rows, shape, index, nbr=None):
    """Returns (nbr [rows_cap, 27], tile_mask [tiles])."""
    D, H, W = shape
    rows_cap = coors.shape[0]
    if nbr is None:
        nbr = torch.empty((rows_cap, 27), dtype=torch.int32, device=coors.device)
    tmask = _tile_mask_buffer(rows_cap, coors.device)
    _call("sassd_rulebook_subm", None, _ptr(coors), _ptr(d_rows), rows_cap, D, H, W, _ptr(index.keys), _ptr(index.vals),
                                   index.slots, _ptr(nbr), _ptr(tmask), _stream())
    return nbr, tmask


def conv_out_shape(shape):
    return [(s + 2 - 3) // 2 + 1 for s in shape]


def rulebook_conv_outputs(coors_in, d_rows_in, batch, shape, rows_cap_out, status, ws=None, ws_key="rbconv",
                          index_out=None):
    """Active output set of a strided (k3,s2,p1) conv, sorted by flattened index.  With ``index_out`` (a fresh
    HashIndex of the output level) the rows are hashed as they are emitted.  Returns coors_out [cap,4], d_rows_out [1],
    out_shape."""
    dev = coors_in.device
    D, H, W = shape
    Do, Ho, Wo = conv_out_shape(shape)
    coors_out = torch.empty((rows_cap_out, 4), dtype=torch.int32, device=dev)
    d_rows_out = torch.empty((1,), dtype=torch.int32, device=dev)
    nbytes = _L().sassd_rulebook_conv_workspace_bytes(batch, Do, Ho, Wo)
    w = (ws or _WS).get(ws_key, nbytes, dev)
    if index_out is None:
        _call("sassd_rulebook_conv_outputs", None, _ptr(coors_in), _ptr(d_rows_in), coors_in.shape[0], batch, D, H, W,
              _ptr(coors_out), _ptr(d_rows_out), rows_cap_out, _ptr(status), _ptr(w), w.numel(), _stream())
    else:
        _call("sassd_rulebook_conv_outputs_hash", None, _ptr(coors_in), _ptr(d_rows_in), coors_in.shape[0], batch, D, H, W,
              _ptr(coors_out), _ptr(d_rows_out), rows_cap_out, _ptr(index_out.keys), _ptr(index_out.vals),
              index_out.slots, _ptr(status), _ptr(w), w.numel(), _stream())
    return coors_out, d_rows_out, [Do, Ho, Wo]


def rulebook_conv_nbr(coors_out, d_rows_out, shape_in, index_in):
    """Neighbour table of the strided conv (probes the INPUT level's hash).  Returns nbr [cap,27], tile_mask."""
    D, H, W = shape_in
    rows_cap_out = coors_out.shape[0]
    nbr = torch.empty((rows_cap_out, 27), dtype=torch.int32, device=coors_out.device)
    tmask = _tile_mask_buffer(rows_cap_out, coors_out.device)
    _call("sassd_rulebook_conv_nbr", None, _ptr(coors_out), _ptr(d_rows_out), rows_cap_out, D, H, W, _ptr(index_in.keys),
          _ptr(index_in.vals), index_in.slots, _ptr(nbr), _ptr(tmask), _stream())
    return nbr, tmask


def rulebook_conv(coors_in, d_rows_in, batch, shape, index_in, rows_cap_out, status, ws=None, ws_key="rbconv",
                  index_out=None):
    """Strided (k3,s2,p1) rulebook.  Returns coors_out [cap,4], d_rows_out [1], nbr [cap,27], out_shape, tile_mask."""
    coors_out, d_rows_out, so = rulebook_conv_outputs(coors_in, d_rows_in, batch, shape, rows_cap_out, status, ws, ws_key,
                                                      index_out)
    nbr, tmask = rulebook_conv_nbr(coors_out, d_rows_out, shape, index_in)
    return coors_out, d_rows_out, nbr, so, tmask


def rulebook_pairs(nbr, d_rows):
    rows_cap = nbr.shape[0]
    pairs = torch.empty((2, 27, rows_cap), dtype=torch.int32, device=nbr.device)
    num = torch.empty((27,), dtype=torch.int32, device=nbr.device)
    _call("sassd_rulebook_pairs", None, _ptr(nbr), _ptr(d_rows), rows_cap, _ptr(pairs), _ptr(num), _stream())
    return pairs, num


# ---------------------------------------------------------------------------- gathered conv
_TC_PACKS = {}
# Bumped by every fill of the dense conv's caches (weight pack, constant vector, background), each of which queues work
# on the stream: conv2d_split sees from it whether its preparation launched anything after the input's producer.
_CONV2D_FILLS = 0


def check_f16_weight(weight, what):
    """Refuse a weight the 3xFP16 split cannot hold: |w| >= 65520 would pack as hi = +-inf, lo = -+inf and turn every
    output of the layer into NaN.  One host read per pack (packs are made once per load, before any capture)."""
    if weight.numel() == 0:
        return
    m = float(weight.detach().abs().max())     # a NaN weight passes (NaN >= x is false): the convs propagate it
    if m >= _lib.F16_SPLIT_MAX:
        raise ValueError("%s: weight magnitude %g is out of the 3xFP16 split's range (|w| < 65520); run the layer at "
                         "PREC_FP32" % (what, m))


def pack_tc(weight, precision):
    """weight [taps, cin, cout] fp32 (device) -> tensor-core pack (hi/lo split, 128B-swizzled K-major blocks)."""
    taps, cin, cout = weight.shape
    nbytes = _L().sassd_gconv_pack_bytes(taps, cin, cout, precision)
    packed = torch.empty((nbytes,), dtype=torch.uint8, device=weight.device)
    _call("sassd_gconv_pack", None, _ptr(weight), taps, cin, cout, precision, _ptr(packed), _stream())
    return packed


def tc_pack_cached(weight, precision):
    """Pack once per weight tensor.  The entry keeps the source tensor alive so that its address cannot be
    recycled for a different weight while the pack is cached (bounded FIFO)."""
    key = (weight.data_ptr(), weight._version, tuple(weight.shape), precision)
    ent = _TC_PACKS.get(key)
    if ent is None:
        if precision == PREC_F16X3:
            taps, cin, cout = weight.shape
            check_f16_weight(weight, "gconv[taps=%d %d->%d]" % (taps, cin, cout))
        if len(_TC_PACKS) >= 256:
            _TC_PACKS.pop(next(iter(_TC_PACKS)))
        ent = (pack_tc(weight.contiguous(), precision), weight)
        _TC_PACKS[key] = ent
    return ent[0]


def conv2d_pack_cached(weight):
    """Weight pack of sassd_conv2d_f16x3 (cached like tc_pack_cached): wgmma register fragments for cout > 64, the
    F16X3 tensor-core pack otherwise."""
    key = (weight.data_ptr(), weight._version, tuple(weight.shape), "conv2d")
    ent = _TC_PACKS.get(key)
    if ent is None:
        if len(_TC_PACKS) >= 256:
            _TC_PACKS.pop(next(iter(_TC_PACKS)))
        w = weight.contiguous()
        taps, cin, cout = w.shape
        check_f16_weight(w, "conv2d_tma[taps=%d %d->%d]" % (taps, cin, cout))
        nbytes = _L().sassd_conv2d_pack_bytes(taps, cin, cout)
        if nbytes == 0:
            raise _lib.SassdError("sassd_conv2d_pack_bytes: unsupported shape taps=%d cin=%d cout=%d" % (taps, cin, cout))
        packed = torch.empty((nbytes,), dtype=torch.uint8, device=w.device)
        _call("sassd_conv2d_pack", None, _ptr(w), taps, cin, cout, _ptr(packed), _stream())
        ent = (packed, weight)
        _TC_PACKS[key] = ent
        global _CONV2D_FILLS
        _CONV2D_FILLS += 1
    return ent[0]


def spconv_pack_cached(weight, cin_stored):
    """Tap-packed fp16 hi/lo weight blocks for sassd_spconv_f16x3 (cached like tc_pack_cached)."""
    key = (weight.data_ptr(), weight._version, tuple(weight.shape), "spconv", cin_stored)
    ent = _TC_PACKS.get(key)
    if ent is None:
        if len(_TC_PACKS) >= 256:
            _TC_PACKS.pop(next(iter(_TC_PACKS)))
        w = weight.contiguous()
        taps, cin, cout = w.shape
        check_f16_weight(w, "spconv_split[taps=%d %d->%d]" % (taps, cin, cout))
        nbytes = _L().sassd_spconv_pack_bytes(taps, cin_stored, cout)
        if nbytes == 0:
            raise _lib.SassdError("sassd_spconv_pack_bytes: unsupported shape taps=%d cin_stored=%d cout=%d"
                             % (taps, cin_stored, cout))
        packed = torch.empty((nbytes,), dtype=torch.uint8, device=w.device)
        _call("sassd_spconv_pack", None, _ptr(w), taps, cin, cin_stored, cout, _ptr(packed), _stream())
        ent = (packed, weight)
        _TC_PACKS[key] = ent
    return ent[0]


def gconv(inp, weight, scale, shift, out, *, mode, taps, cin, cout, relu, nbr=None, d_rows=None, rows_cap=None,
          batch=0, H=0, W=0, precision=PREC_FP32, status=None):
    """out[m,:] = act((sum_t in[row(m,t),:] @ W[t]) * scale + shift); see sassd_b200.h.  ``status``: the step's status
    word, F16_RANGE when PREC_F16X3 meets an input it cannot split."""
    if precision in (PREC_TF32X3, PREC_F16X3):
        weight = tc_pack_cached(weight, precision)
    d = GConvDesc()
    d.mode, d.precision = mode, precision
    d.cin, d.cout, d.taps = cin, cout, taps
    d.in_stride = inp.stride(-2) if inp.dim() >= 2 else cin
    d.out_stride = out.stride(-2) if out.dim() >= 2 else cout
    d.rows_cap = int(rows_cap if rows_cap is not None else out.numel() // d.out_stride)
    d.batch, d.H, d.W = batch, H, W
    d.relu = 1 if relu else 0
    label = "gconv[%s taps=%d %d->%d]" % (("table", "conv2d", "rows")[mode], taps, cin, cout)
    _call("sassd_gconv_status", label, ctypes.byref(d), _ptr_any(inp), _ptr(weight), _ptr(scale), _ptr(shift), _ptr(nbr),
                           _ptr(d_rows), _ptr_any(out), _ptr(status), _stream())
    return out


def _ptr_any(t):
    assert t.is_cuda
    return ctypes.c_void_p(t.data_ptr())


def sparse_to_bev(feat, coors, d_rows, C, D, H, W, bev):
    _call("sassd_sparse_to_bev", None, _ptr(feat), _ptr(coors), _ptr(d_rows), feat.shape[0], C, D, H, W, _ptr(bev),
                                   _stream())
    return bev


# ---------------------------------------------------------------------------- head tail
def decode_select(head, num_class, anchors, mask, thr, k_cap, status, ws=None):
    """head [B,H,W,stride] NHWC; anchors [Na,7] (shared) or [B,Na,7] (per frame).
    Returns boxes [B,k_cap,7], labels, index, d_k [B]."""
    dev = head.device
    B, H, W, stride = head.shape
    per_frame = 1 if anchors.dim() == 3 else 0
    assert not per_frame or anchors.shape[0] == B
    na = anchors.shape[-2]
    boxes = torch.empty((B, k_cap, 7), dtype=torch.float32, device=dev)
    labels = torch.empty((B, k_cap), dtype=torch.int32, device=dev)
    index = torch.empty((B, k_cap), dtype=torch.int32, device=dev)
    d_k = torch.empty((B,), dtype=torch.int32, device=dev)
    nbytes = _L().sassd_decode_select_workspace_bytes(B, na)
    w = (ws or _WS).get("decode", nbytes, dev)
    _call("sassd_decode_select", None, _ptr(head), stride, B, H, W, num_class, _ptr(anchors), per_frame, _ptr(mask), na,
                                   ctypes.c_float(thr), _ptr(boxes), _ptr(labels), _ptr(index), _ptr(d_k), k_cap,
                                   _ptr(status), _ptr(w), w.numel(), _stream())
    return boxes, labels, index, d_k


def pswarp(feat, boxes, d_k, off_x, off_y, spatial_scale):
    B, H, W, stride = feat.shape
    k_cap = boxes.shape[1]
    scores = torch.empty((B, k_cap), dtype=torch.float32, device=feat.device)
    _call("sassd_pswarp", None, _ptr(feat), stride, B, H, W, _ptr(boxes), _ptr(d_k), k_cap, ctypes.c_float(off_x),
                            ctypes.c_float(off_y), ctypes.c_float(spatial_scale), _ptr(scores), _stream())
    return scores


def rescore_nms(boxes, scores, labels, d_k, score_thr, iou_thr, det_cap, status, ws=None):
    dev = boxes.device
    B, k_cap = boxes.shape[0], boxes.shape[1]
    det = torch.empty((B, det_cap, 9), dtype=torch.float32, device=dev)
    d_ndet = torch.empty((B,), dtype=torch.int32, device=dev)
    nbytes = _L().sassd_rescore_nms_workspace_bytes(B, k_cap, NMS_CAP)
    w = (ws or _WS).get("nms", nbytes, dev)
    _call("sassd_rescore_nms", None, _ptr(boxes), _ptr(scores), _ptr(labels), _ptr(d_k), B, k_cap,
                                 ctypes.c_float(score_thr), ctypes.c_float(iou_thr), NMS_CAP, _ptr(det), _ptr(d_ndet),
                                 det_cap, _ptr(status), _ptr(w), w.numel(), _stream())
    return det, d_ndet


def kitti_format(det, d_ndet, meta):
    """det [B,det_cap,9] f32, d_ndet [B] i32 (rescore_nms), meta [B,36] f64 (results.meta_block; device).
    Returns (rows [B,det_cap,14] f64, n_out [B] i32): per frame the KITTI annotation rows of the detections whose image
    projection is not wholly outside the image (results.annos_from_rows), in detection order.  Rows past n_out[b] are
    left unwritten."""
    dev = det.device
    B, det_cap = det.shape[0], det.shape[1]
    assert meta.dtype == torch.float64 and tuple(meta.shape) == (B, _lib.KITTI_META), "meta must be float64 [B,36]"
    rows = torch.empty((B, det_cap, _lib.KITTI_ROW), dtype=torch.float64, device=dev)
    n_out = torch.empty((B,), dtype=torch.int32, device=dev)
    _call("sassd_kitti_format", None, _ptr(det), _ptr(d_ndet), B, det_cap, _ptr(meta), _ptr(rows), _ptr(n_out),
          _stream())
    return rows, n_out


def kitti_eval_flags(gt_name, gt_occ, gt_trunc, gt_bbox, dt_name, dt_bbox, classes, limits):
    """clean_data's ignore flags on the device (csrc/kitti_match.cu).  gt_name / dt_name [rows] i32 name ids, gt_occ /
    gt_trunc [G] f64, gt_bbox / dt_bbox [rows,4] f64, classes [C,2] i32 (name id, ignored name id or -1), limits
    [Dn,3] f64 (max occlusion, max truncation, min height).  Returns (ign_gt [C,Dn,G] i8, ign_dt [C,Dn,D] i8,
    n_valid [C,Dn] i32)."""
    dev = gt_bbox.device
    G, D, C, Dn = gt_name.shape[0], dt_name.shape[0], classes.shape[0], limits.shape[0]
    ign_gt = torch.empty((C, Dn, G), dtype=torch.int8, device=dev)
    ign_dt = torch.empty((C, Dn, D), dtype=torch.int8, device=dev)
    n_valid = torch.zeros((C, Dn), dtype=torch.int32, device=dev)
    _call("sassd_kitti_eval_flags", None, G, _ptr(gt_name), _ptr(gt_occ), _ptr(gt_trunc), _ptr(gt_bbox), D,
          _ptr(dt_name), _ptr(dt_bbox), C, _ptr(classes), Dn, _ptr(limits), _ptr(ign_gt), _ptr(ign_dt), _ptr(n_valid),
          _stream())
    return ign_gt, ign_dt, n_valid


def kitti_eval_flags_ranged(gt_name, gt_occ, gt_trunc, gt_bbox, gt_cam, dt_name, dt_bbox, dt_cam, classes, limits,
                            ranges):
    """kitti_eval_flags with a range bin per difficulty entry (csrc/kitti_match.cu): gt_cam / dt_cam [rows,7] f64
    camera rows, ranges [Dn,2] f64 (lo, hi) or None (no range test; an entry whose lo is -inf has none either).
    Returns (ign_gt, ign_dt, n_valid, gt_range [G] f64, dt_range [D] f64): the flags and every row's ground distance
    sqrt(x * x + z * z)."""
    dev = gt_bbox.device
    G, D, C, Dn = gt_name.shape[0], dt_name.shape[0], classes.shape[0], limits.shape[0]
    ign_gt = torch.empty((C, Dn, G), dtype=torch.int8, device=dev)
    ign_dt = torch.empty((C, Dn, D), dtype=torch.int8, device=dev)
    n_valid = torch.zeros((C, Dn), dtype=torch.int32, device=dev)
    gt_range = torch.empty((G,), dtype=torch.float64, device=dev)
    dt_range = torch.empty((D,), dtype=torch.float64, device=dev)
    _call("sassd_kitti_eval_flags_ranged", None, G, _ptr(gt_name), _ptr(gt_occ), _ptr(gt_trunc), _ptr(gt_bbox),
          _ptr(gt_cam), D, _ptr(dt_name), _ptr(dt_bbox), _ptr(dt_cam), C, _ptr(classes), Dn, _ptr(limits),
          _ptr(ranges) if ranges is not None else None, _ptr(ign_gt), _ptr(ign_dt), _ptr(n_valid), _ptr(gt_range),
          _ptr(dt_range), _stream())
    return ign_gt, ign_dt, n_valid, gt_range, dt_range


def kitti_eval_overlaps(nsets, nframes, gt_off, dt_off, ov_off, gt_cam, dt_cam, gt_bbox, dt_bbox, bev_iou, bev_inter,
                        total_pairs, max_pairs):
    """The bbox, BEV and 3-D overlap matrices (f64 [total_pairs], blocks at ov_off) of every (set, frame) block: gt_cam /
    dt_cam [rows,7] f64 camera boxes, bev_iou / bev_inter the rotated overlaps at criterion -1 / 2 (f32, same blocks)."""
    out = [torch.empty((max(int(total_pairs), 1),), dtype=torch.float64, device=gt_cam.device) for _ in range(3)]
    _call("sassd_kitti_eval_overlaps", None, nsets, nframes, _ptr(gt_off), _ptr(dt_off), _ptr(ov_off), _ptr(gt_cam),
          _ptr(dt_cam), _ptr(gt_bbox), _ptr(dt_bbox), _ptr(bev_iou), _ptr(bev_inter), int(max_pairs), _ptr(out[0]),
          _ptr(out[1]), _ptr(out[2]), _stream())
    return out


def kitti_eval_match(desc, njobs, score_total, ws=None):
    """Pass 1, thresholds and pass 2 of the KITTI matching for every job of ``desc`` (lib.KittiEvalDesc whose pointers
    are device tensors the caller keeps alive).  Returns (thresholds [njobs,41] f64, n_thresh [njobs] i32,
    pr [njobs,41,4] f64)."""
    dev = torch.device("cuda", torch.cuda.current_device())
    scores = torch.empty((max(int(score_total), 1),), dtype=torch.float64, device=dev)
    n_scores = torch.empty((njobs,), dtype=torch.int32, device=dev)
    thresholds = torch.zeros((njobs, 41), dtype=torch.float64, device=dev)
    n_thresh = torch.empty((njobs,), dtype=torch.int32, device=dev)
    pr = torch.empty((njobs, 41, 4), dtype=torch.float64, device=dev)
    nbytes = _L().sassd_kitti_eval_workspace_bytes(desc.max_nd, desc.max_ng)
    w = (ws or _WS).get("kitti_eval", nbytes, dev)
    _call("sassd_kitti_eval_match", None, ctypes.byref(desc), _ptr(scores), _ptr(n_scores), _ptr(thresholds),
          _ptr(n_thresh), _ptr(pr), _ptr(w), w.numel(), _stream())
    return thresholds, n_thresh, pr


def kitti_eval_assign(desc, row, ndiff, gt_cam, dt_cam, ws=None):
    """The match table of the first ``ndiff`` difficulty entries of ``desc`` at min-overlap row ``row`` (csrc/
    kitti_match.cu).  Returns (gt_det [K,C,ndiff,3,G] i32, gt_ov [K,C,ndiff,3,G] f64, dt_state [C,ndiff,3,D] i8,
    tp_err [K,C,ndiff,G,3] f64)."""
    dev = gt_cam.device
    K, C, G, D = desc.nsets, desc.nclass, gt_cam.shape[0], dt_cam.shape[0]
    gt_det = torch.empty((K, C, ndiff, 3, G), dtype=torch.int32, device=dev)
    gt_ov = torch.empty((K, C, ndiff, 3, G), dtype=torch.float64, device=dev)
    dt_state = torch.empty((C, ndiff, 3, D), dtype=torch.int8, device=dev)
    tp_err = torch.empty((K, C, ndiff, G, 3), dtype=torch.float64, device=dev)
    w = (ws or _WS).get("kitti_eval", _L().sassd_kitti_eval_workspace_bytes(desc.max_nd, desc.max_ng), dev)
    _call("sassd_kitti_eval_assign", None, ctypes.byref(desc), int(row), int(ndiff), _ptr(gt_cam), _ptr(dt_cam),
          _ptr(gt_det), _ptr(gt_ov), _ptr(dt_state), _ptr(tp_err), _ptr(w), w.numel(), _stream())
    return gt_det, gt_ov, dt_state, tp_err


def kitti_scan_labels(buf, file_off):
    """buf [bytes] u8: every file's bytes back to back, file f at [file_off[f], file_off[f+1]) (file_off [F+1] i64;
    device).  Returns (n_lines [F] i32, flags [F] i32 of lib.KITTI_PARSE_DEFER / KITTI_PARSE_SCORE), csrc/kitti_parse.cu:
    a deferred file is outside the device grammar and is read on the host."""
    F = file_off.shape[0] - 1
    n_lines = torch.empty((F,), dtype=torch.int32, device=buf.device)
    flags = torch.empty((F,), dtype=torch.int32, device=buf.device)
    _call("sassd_kitti_scan_labels", None, _ptr(buf), _ptr(file_off), F, _ptr(n_lines), _ptr(flags), _stream())
    return n_lines, flags


def kitti_parse_labels(buf, file_off, flags, row_off, nrows, names, name_off, ws=None):
    """The rows of every file kitti_scan_labels did not defer, file f's lines at rows row_off[f] .. (row_off [F+1] i32;
    names / name_off: the lower-cased class-name table, u8 bytes and [N+1] i32 offsets).  Returns the columns
    (name_id [R] i32, dontcare [R] i32, truncated, occluded, alpha [R] f64, bbox [R,4] f64, cam [R,7] f64, score [R]
    f64); a deferred file's rows are left unwritten."""
    dev = buf.device
    F = file_off.shape[0] - 1
    f64 = dict(dtype=torch.float64, device=dev)
    out = [torch.empty((nrows,), dtype=torch.int32, device=dev), torch.empty((nrows,), dtype=torch.int32, device=dev),
           torch.empty((nrows,), **f64), torch.empty((nrows,), **f64), torch.empty((nrows,), **f64),
           torch.empty((nrows, 4), **f64), torch.empty((nrows, 7), **f64), torch.empty((nrows,), **f64)]
    w = (ws or _WS).get("kitti_parse", _L().sassd_kitti_parse_workspace_bytes(nrows), dev)
    _call("sassd_kitti_parse_labels", None, _ptr(buf), _ptr(file_off), F, _ptr(flags), _ptr(row_off), nrows,
          _ptr(names), _ptr(name_off), name_off.shape[0] - 1, *[_ptr(t) for t in out], _ptr(w), w.numel(), _stream())
    return out


def merge_detections(dets, label_offsets):
    """dets: per member (det [B,cap_m,9] f32, d_ndet [B] i32) as rescore_nms returns them; label_offsets: per member
    the index of its first class in the merged class list.  Returns (det [B,sum cap_m,9], d_ndet [B]): per frame the
    members' rows in member order, labels offset (csrc/merge.cu).  Rows past d_ndet[b] are left unwritten."""
    M = len(dets)
    assert 1 <= M <= _lib.MERGE_MAX and len(label_offsets) == M, "1..%d members, one label offset each" % _lib.MERGE_MAX
    B = dets[0][0].shape[0]
    for d, n in dets:
        assert d.dtype == torch.float32 and d.dim() == 3 and d.shape[0] == B and d.shape[2] == 9 and d.is_contiguous()
        assert n.dtype == torch.int32 and tuple(n.shape) == (B,)
    caps = [int(d.shape[1]) for d, _ in dets]
    det = torch.empty((B, sum(caps), 9), dtype=torch.float32, device=dets[0][0].device)
    d_ndet = torch.empty((B,), dtype=torch.int32, device=det.device)
    _call("sassd_merge_detections", None, (ctypes.c_void_p * M)(*[_ptr(d) for d, _ in dets]),
          (ctypes.c_void_p * M)(*[_ptr(n) for _, n in dets]), (ctypes.c_int * M)(*caps),
          (ctypes.c_int * M)(*[int(o) for o in label_offsets]), M, B, _ptr(det), _ptr(d_ndet), _stream())
    return det, d_ndet


# ---------------------------------------------------------------------------- auxiliary point-wise head
def three_nn(mean, coors0, d_rows0, levels, points_mean=False):
    """mean [cap0,4] f32 (x, y, z, r of each voxel), coors0 [cap0,4] i32 (b,z,y,x), d_rows0 [1]; ``levels``: three
    (coors [capL,4] i32, d_rows [1]) of backbone levels 1..3, rows sorted by flattened (b,z,y,x).  Returns
    (idx [cap0,3,3] i32, dist2 [cap0,3,3] f32, points_mean [cap0,4] f32 or None): per voxel row, level and k the global
    row of its k-th nearest centre of the same frame and the squared distance (pointnet2 three_nn, bit for bit;
    missing slots idx 0, dist2 +inf); points_mean rows are (b, x, y, z).  Rows past d_rows0 are left unwritten."""
    dev = mean.device
    cap0 = mean.shape[0]
    assert len(levels) == 3 and coors0.shape[0] == cap0 and tuple(mean.shape[1:]) == (4,) and mean.dtype == torch.float32
    idx = torch.empty((cap0, 3, 3), dtype=torch.int32, device=dev)
    dist2 = torch.empty((cap0, 3, 3), dtype=torch.float32, device=dev)
    pm = torch.empty((cap0, 4), dtype=torch.float32, device=dev) if points_mean else None
    (c1, n1), (c2, n2), (c3, n3) = levels
    _call("sassd_three_nn", None, _ptr(mean), _ptr(coors0), _ptr(d_rows0), cap0, _ptr(c1), _ptr(n1), _ptr(c2),
          _ptr(n2), _ptr(c3), _ptr(n3), _ptr(idx), _ptr(dist2), _ptr(pm), _stream())
    return idx, dist2, pm


def point_level(feat=None, split=None, channels=None):
    """Feature rows of one backbone level for point_aux_head: fp32 ``feat`` [cap, >=C] or split fp16 rows ``split``
    [2, cap, >=C] (features_to_split / spconv_split)."""
    d = _lib.PointLevels()
    if feat is not None:
        assert feat.dtype == torch.float32 and feat.dim() == 2
        d.rows, d.plane_stride, d.row_stride, d.split = _ptr(feat).value, 0, feat.stride(0), 0
        d.channels = channels if channels is not None else feat.shape[1]
    else:
        assert split.dtype == torch.float16 and split.dim() == 3 and split.shape[0] == 2
        d.rows, d.plane_stride, d.row_stride, d.split = _ptr(split).value, split.stride(0), split.stride(1), 1
        d.channels = channels if channels is not None else split.shape[2]
    return d


def point_aux_head(idx, dist2, d_rows0, levels, w_fc_t, w_out):
    """idx / dist2 from three_nn; ``levels``: three point_level() of levels 1..3 (32, 64, 64 channels); w_fc_t
    [160,64] = point_fc.weight^T, w_out [4,64] = point_cls.weight then point_reg.weight (fp32, device).
    Returns (cls [cap0] logits, reg [cap0,3]); rows past d_rows0 are left unwritten."""
    dev = idx.device
    cap0 = idx.shape[0]
    assert tuple(w_fc_t.shape) == (_lib.POINT_FC_IN, _lib.POINT_FC_OUT) and tuple(w_out.shape) == (4, _lib.POINT_FC_OUT)
    arr = (_lib.PointLevels * 3)(*levels)
    cls = torch.empty((cap0,), dtype=torch.float32, device=dev)
    reg = torch.empty((cap0, 3), dtype=torch.float32, device=dev)
    _call("sassd_point_aux_head", None, _ptr(idx), _ptr(dist2), _ptr(d_rows0), cap0, arr, _ptr(w_fc_t), _ptr(w_out),
          _ptr(cls), _ptr(reg), _stream())
    return cls, reg


def nms_mask(boxes5, thr):
    n = boxes5.shape[0]
    colb = (n + 63) // 64
    mask = torch.zeros((n, max(colb, 1)), dtype=torch.int64, device=boxes5.device)
    _call("sassd_nms_mask", None, _ptr(boxes5), n, ctypes.c_float(thr), _ptr(mask), _stream())
    return mask[:, :colb]


def nms_sorted(boxes5, thr):
    """boxes sorted by score.  Returns (keep [n] int64 capacity-sized, d_nkeep [1])."""
    dev = boxes5.device
    n = boxes5.shape[0]
    keep = torch.empty((max(n, 1),), dtype=torch.int64, device=dev)
    d_n = torch.zeros((1,), dtype=torch.int32, device=dev)
    nbytes = _L().sassd_nms_workspace_bytes(n)
    w = _WS.get("nms_sorted", nbytes, dev)
    _call("sassd_nms_sorted", None, _ptr(boxes5), n, ctypes.c_float(thr), _ptr(keep), _ptr(d_n), _ptr(w), w.numel(),
                                _stream())
    return keep, d_n


def boxes_iou_bev(a, b):
    out = torch.empty((a.shape[0], b.shape[0]), dtype=torch.float32, device=a.device)
    _call("sassd_boxes_iou_bev", None, _ptr(a), a.shape[0], _ptr(b), b.shape[0], _ptr(out), _stream())
    return out


# ---------------------------------------------------------------------------- training targets and losses
# Output vector of loss_vector(): the keys of SingleStageDetector.forward_train, in this order.
LOSS_KEYS = ("aux_loss_cls", "aux_loss_reg", "rpn_loc_loss", "rpn_cls_loss", "rpn_dir_loss", "loss_cls")


def _loss_ws(batch, gt_cap, device, ws=None):
    nbytes = _L().sassd_loss_workspace_bytes(batch, gt_cap)
    return (ws or _WS).get("loss", nbytes, device)


def points_in_boxes(points_mean, d_rows, gt, d_ngt, status, ws=None):
    """points_mean [cap,4] (b, x, y, z), d_rows [1]; gt [B,gt_cap,7] (x, y, z_bottom, w, l, h, ry), d_ngt [B] i32.
    Returns (labels [cap] i32, offsets [cap,3], d_npos [1]): pts_in_boxes3d per frame (build_aux_target).  Rows past
    d_rows are left unwritten."""
    dev = points_mean.device
    cap = points_mean.shape[0]
    B, gt_cap = gt.shape[0], gt.shape[1]
    labels = torch.empty((cap,), dtype=torch.int32, device=dev)
    offsets = torch.empty((cap, 3), dtype=torch.float32, device=dev)
    d_npos = torch.empty((1,), dtype=torch.int32, device=dev)
    _call("sassd_points_in_boxes", None, _ptr(points_mean), _ptr(d_rows), cap, _ptr(gt), _ptr(d_ngt), B, gt_cap,
          _ptr(labels), _ptr(offsets), _ptr(d_npos), _ptr(status), _stream())
    return labels, offsets, d_npos


def assign_rpn(anchors, mask, num_class, gt, gt_class, gt_label, d_ngt, pos_thr, neg_thr, status, ws=None):
    """anchors [Na,7] (shared) or [B,Na,7], classes concatenated; mask [B,Na] u8; gt [B,gt_cap,7], gt_class /
    gt_label [B,gt_cap] i32, d_ngt [B]; pos_thr / neg_thr one per class.  Returns (labels [B,Na] i32, targets
    [B,Na,7], ious [B,Na], d_npos [B])."""
    dev = gt.device
    B, gt_cap = gt.shape[0], gt.shape[1]
    na = anchors.shape[-2]
    labels = torch.empty((B, na), dtype=torch.int32, device=dev)
    targets = torch.empty((B, na, 7), dtype=torch.float32, device=dev)
    ious = torch.empty((B, na), dtype=torch.float32, device=dev)
    d_npos = torch.empty((B,), dtype=torch.int32, device=dev)
    pos = (ctypes.c_float * num_class)(*[float(v) for v in pos_thr])
    neg = (ctypes.c_float * num_class)(*[float(v) for v in neg_thr])
    w = _loss_ws(B, gt_cap, dev, ws)
    _call("sassd_assign_rpn", None, _ptr(anchors), 1 if anchors.dim() == 3 else 0, _ptr(mask), na, num_class, _ptr(gt),
          _ptr(gt_class), _ptr(gt_label), _ptr(d_ngt), B, gt_cap, pos, neg, _ptr(labels), _ptr(targets), _ptr(ious),
          _ptr(d_npos), _ptr(status), _ptr(w), w.numel(), _stream())
    return labels, targets, ious, d_npos


def assign_pswarp(gt, d_ngt, boxes, d_k, pos_thr, neg_thr, status, d_head=None, head_cap=0, ws=None):
    """gt [B,gt_cap,7], d_ngt [B]; boxes [B,n,7]: slots [0, head_cap) hold d_head[b] boxes, slots [head_cap, n) hold
    d_k[b] boxes.  Returns (labels [B,n] i32 (-1 in empty slots), ious [B,n], d_npos [B])."""
    dev = gt.device
    B, gt_cap = gt.shape[0], gt.shape[1]
    n = boxes.shape[1]
    labels = torch.empty((B, n), dtype=torch.int32, device=dev)
    ious = torch.empty((B, n), dtype=torch.float32, device=dev)
    d_npos = torch.empty((B,), dtype=torch.int32, device=dev)
    w = _loss_ws(B, gt_cap, dev, ws)
    _call("sassd_assign_pswarp", None, _ptr(gt), _ptr(d_ngt), B, gt_cap, _ptr(boxes), n, _ptr(d_head), head_cap,
          _ptr(d_k), ctypes.c_float(pos_thr), ctypes.c_float(neg_thr), _ptr(labels), _ptr(ious), _ptr(d_npos),
          _ptr(status), _ptr(w), w.numel(), _stream())
    return labels, ious, d_npos


def rpn_loss(head, num_class, anchors, labels, targets, d_npos, out, ws=None):
    """head [B,H,W,stride] (SSDRotateHead.forward_nhwc); writes out[0:3] = rpn_loc_loss, rpn_cls_loss, rpn_dir_loss."""
    B, H, W, stride = head.shape
    w = _loss_ws(B, 1, head.device, ws)
    _call("sassd_rpn_loss", None, _ptr(head), stride, B, H, W, num_class, _ptr(anchors), 1 if anchors.dim() == 3 else 0,
          anchors.shape[-2], _ptr(labels), _ptr(targets), _ptr(d_npos), _ptr(out), _ptr(w), w.numel(), _stream())


def pswarp_loss(scores, labels, d_npos, out, ws=None):
    """scores / labels [B,n]; writes out[0] = loss_cls."""
    B, n = scores.shape
    w = _loss_ws(B, 1, scores.device, ws)
    _call("sassd_pswarp_loss", None, _ptr(scores), _ptr(labels), B, n, _ptr(d_npos), _ptr(out), _ptr(w), w.numel(),
          _stream())


def aux_loss(point_cls, point_reg, labels, offsets, d_rows, batch, d_npos, out, ws=None):
    """writes out[0:2] = aux_loss_cls, aux_loss_reg."""
    cap = point_cls.shape[0]
    w = _loss_ws(batch, 1, point_cls.device, ws)
    _call("sassd_aux_loss", None, _ptr(point_cls), _ptr(point_reg), _ptr(labels), _ptr(offsets), _ptr(d_rows), cap,
          batch, _ptr(d_npos), _ptr(out), _ptr(w), w.numel(), _stream())


# ---------------------------------------------------------------------------- TMA dense conv on split maps
class SplitMap:
    """Activation map as two fp16 planes [2, B, H, W, C_stored] (hi, lo*2048) — the operand format of
    sassd_conv2d_f16x3; ``channels`` of the C_stored are meaningful, the rest are zero."""

    def __init__(self, planes, channels, tile_dist=None, reach=0, const=None, background=None, status=None):
        # Maps that descend from a scattered sparse tensor are constant over large regions.  tile_dist: int32
        # [B * tiles_y * tiles_x], pixel distance of every conv tile to the nearest active cell of the scattered map;
        # reach: number of 3x3 convs applied since; const: fp32 [channels] value of the constant region (None = 0);
        # background: SplitMap of batch 1, the same layers applied to an empty scene (None: all zero at reach 0,
        # unknown beyond).  conv2d_split uses them to skip the tiles whose output is the layer's constant or, on the
        # image border, the layer's background (see sassd_conv2d_f16x3_occ_bg).
        self.planes, self.channels = planes, channels
        self.tile_dist, self.reach, self.const = tile_dist, reach, const
        self.background = background
        # status: the step's int32 status word, which every conv on this map and the maps derived from it flags
        # F16_RANGE in when a value it stores overflows the split (None: unchecked)
        self.status = status

    @property
    def shape(self):
        return (self.planes.shape[1], self.planes.shape[2], self.planes.shape[3], self.channels)

    @property
    def device(self):
        return self.planes.device

    def float(self):
        """fp32 NHWC reconstruction (hi + lo/2048), for API-compat consumers and tests."""
        return (self.planes[0].float() + self.planes[1].float() * (1.0 / 2048.0))[..., : self.channels].contiguous()

    @staticmethod
    def from_float(x):
        """Test / compat helper: split an fp32 NHWC map with the same arithmetic as the kernels."""
        B, H, W, C = x.shape
        cs = (C + 63) // 64 * 64
        hi = x.half()
        lo = ((x - hi.float()) * 2048.0).half()
        planes = torch.zeros((2, B, H, W, cs), dtype=torch.float16, device=x.device)
        planes[0, ..., :C] = hi
        planes[1, ..., :C] = lo
        return SplitMap(planes, C)


TILE_OCCUPANCY = os.environ.get("SASSD_TMA_OCC", "1") != "0"     # constant-region tile skipping in the BEV convs
CONV2D_TILE_ORDER = 0       # 1 while a latency-oriented step is captured (computed tiles first, see sassd_b200.h)
CONV2D_COUNTERS = None     # bench instrumentation: {label: int32[2] device tensor} += tiles computed, += tiles
# Per-tile ready counters between consecutive BN = 128 convs launched as programmatic dependents (tile_ready_arena):
# a conv starts each tile once the tiles it reads are stored instead of waiting for the whole previous layer.  Results
# are the same bit for bit either way; SASSD_TILE_FLAGS=0 turns them off for bisecting.
CONV2D_TILE_FLAGS = os.environ.get("SASSD_TILE_FLAGS", "1") != "0"
# Frames per step up to which the counters are used.  At batch 1 a 256-channel layer is about two units per SM and its
# second half mostly idle; at batch 16 it is ~23 units per SM, the tail is small and the per-unit release fences cost
# more than the early starts return (H100 80GB HBM3, 700 W: batch 1 +6 %, batch 16 -2 % with the counters).
TILE_FLAGS_MAX_BATCH = 1
_TILE_FAR = 1 << 20


def _tile_dist(batch, H, W, device):
    if not TILE_OCCUPANCY:
        return None
    th, tw = _lib.CONV2D_TILE_H, _lib.CONV2D_TILE_W
    return torch.full((batch * ((H + th - 1) // th) * ((W + tw - 1) // tw),), _TILE_FAR, dtype=torch.int32, device=device)


def tile_skipping_valid(H, W, reach):
    """Conditions under which the constant-region rule of sassd_conv2d_f16x3_occ is exact.  (a) tile distances are
    only recorded up to SASSD_TILE_DIST_MAX pixels, so a layer further than that from the scattered map cannot tell
    "far" from "just out of range".  (b) zero padding disturbs the constant up to reach-1 pixels from the image edge
    and the kernel exempts only the outermost tile row / column: those edge tiles must be at least that deep, which
    fails for a thin partial last tile (H % 8 or W % 16 small).  The C entry point checks the same and returns
    SASSD_ERR_UNSUPPORTED; here the layer simply falls back to computing every tile."""
    th, tw = _lib.CONV2D_TILE_H, _lib.CONV2D_TILE_W
    if reach > _lib.TILE_DIST_MAX:
        return False
    last_h = H - (H - 1) // th * th
    last_w = W - (W - 1) // tw * tw
    return min(last_h, last_w, th, tw) >= reach - 1


_CONV_CONSTS = {}


def conv_constant(x_const, cin, weight, scale, shift, relu, cout):
    """Output of a conv layer on a constant input map: fp32 [cout], obtained by running the very kernel on a
    3x3-tile map filled with the constant and reading an interior pixel, so tiles that skip the computation store
    bit-identical values.  Depends on weights only (cached; warm before CUDA-graph capture)."""
    key = (weight.data_ptr(), weight._version, None if scale is None else (scale.data_ptr(), scale._version),
           None if shift is None else (shift.data_ptr(), shift._version), bool(relu), cout, cin,
           None if x_const is None else x_const.data_ptr())
    ent = _CONV_CONSTS.get(key)
    if ent is None:
        if len(_CONV_CONSTS) >= 256:
            _CONV_CONSTS.pop(next(iter(_CONV_CONSTS)))
        h, w = 3 * _lib.CONV2D_TILE_H, 3 * _lib.CONV2D_TILE_W
        m = torch.zeros((1, h, w, cin), dtype=torch.float32, device=weight.device)
        if x_const is not None:
            m += x_const[:cin].view(1, 1, 1, cin)
        _, f = conv2d_split(SplitMap.from_float(m), weight, scale, shift, relu, cout, out_split=False, out_f32=True)
        ent = (f[0, h // 2, w // 2, :cout].clone().contiguous(), weight, scale, shift, x_const)   # keep keys alive
        _CONV_CONSTS[key] = ent
        global _CONV2D_FILLS
        _CONV2D_FILLS += 1
    return ent[0]


_BACKGROUNDS = collections.OrderedDict()
# One background is a full map (36 MB for 256 channels on the 200x176 grid, ~0.3 GB for a detector's chain of layers):
# the least recently used are dropped beyond this many bytes, which also bounds the maps a weight reload leaves stale.
BACKGROUND_CACHE_BYTES = 4 << 30
BACKGROUND_PINS = None     # a list while a CUDA graph is captured: the backgrounds its kernels read, kept by the graph


def conv_background(x, weight, scale, shift, relu, cout, out_split, out_f32):
    """The layer's outputs on an empty scene, batch 1: (SplitMap | None, fp32 map | None), computed in full by the very
    kernel from x's background, or None when x's background is unknown.  The border tiles far from every active cell
    copy it (sassd_conv2d_f16x3_occ_bg): their receptive field holds only inactive cells and the zero padding, so they
    equal it bit for bit.  Cached per weights and input background (warm before CUDA-graph capture)."""
    B, H, W, cin = x.shape
    src = x.background
    if src is None and x.reach > 0:
        return None
    key = (weight.data_ptr(), weight._version, None if scale is None else (scale.data_ptr(), scale._version),
           None if shift is None else (shift.data_ptr(), shift._version), bool(relu), cout, cin, x.planes.shape[-1], H, W,
           None if src is None else src.planes.data_ptr(), bool(out_split), bool(out_f32))
    ent = _BACKGROUNDS.get(key)
    if ent is None:
        if src is None:
            src_in = SplitMap(torch.zeros((2, 1, H, W, x.planes.shape[-1]), dtype=torch.float16, device=x.device), cin)
        else:
            src_in = src
        bg = conv2d_split(src_in, weight, scale, shift, relu, cout, out_split=out_split, out_f32=out_f32)
        nbytes = sum(t.numel() * t.element_size() for t in (bg[0] and bg[0].planes, bg[1]) if t is not None)
        ent = (bg, nbytes, weight, scale, shift, src)       # keep the keys alive
        _BACKGROUNDS[key] = ent
        global _CONV2D_FILLS
        _CONV2D_FILLS += 1
        while len(_BACKGROUNDS) > 1 and sum(e[1] for e in _BACKGROUNDS.values()) > BACKGROUND_CACHE_BYTES:
            _BACKGROUNDS.popitem(last=False)
    else:
        _BACKGROUNDS.move_to_end(key)
    if BACKGROUND_PINS is not None:
        BACKGROUND_PINS.append(ent[0])
    return ent[0]


def sparse_to_bev_split(feat, coors, d_rows, C, D, H, W, batch, status=None):
    planes = torch.zeros((2, batch, H, W, D * C), dtype=torch.float16, device=feat.device)
    dist = _tile_dist(batch, H, W, feat.device)
    _call("sassd_sparse_to_bev_split_status", None, _ptr(feat), _ptr(coors), _ptr(d_rows), feat.shape[0], C, D, H, W, batch,
          _ptr(planes), _ptr(dist), _ptr(status), _stream())
    return SplitMap(planes, D * C, dist, status=status)


def tile_ready_arena(x, maps):
    """Ready counters for ``maps`` outputs of a chain of cout > 64 convs on split map x, each conv launched right after
    the one that wrote its input (sassd_conv2d_desc.in_ready / out_ready): a list of int32 [tiles + 1] views of one
    arena, zeroed here, once per call (the arena is a fresh allocation, a node of its own in a captured graph).  None
    when the counters are off: CONV2D_TILE_FLAGS unset, launches not programmatic (without PDL every conv waits for
    the previous one anyway), no status word to report a timed-out wait in, or more than TILE_FLAGS_MAX_BATCH
    frames."""
    B, H, W, _ = x.shape
    if not CONV2D_TILE_FLAGS or x.status is None or B > TILE_FLAGS_MAX_BATCH or not _L().sassd_pdl_enabled():
        return None
    th, tw = _lib.CONV2D_TILE_H, _lib.CONV2D_TILE_W
    n = B * ((H + th - 1) // th) * ((W + tw - 1) // tw) + 1
    return list(torch.zeros((maps, n), dtype=torch.int32, device=x.device).unbind(0))


def conv2d_split(x, weight, scale, shift, relu, cout, out_split=True, out_f32=False, in_ready=None, out_ready=None):
    """x: SplitMap; weight [taps, cin, cout] fp32 (packed on first use).  Returns (SplitMap | None, fp32 map | None).
    in_ready / out_ready (cout > 64): tile_ready_arena counters of x and of the output map.  in_ready requires that
    the launch which wrote x is the last one on the stream before this call; work this call queues itself first (a
    weight pack, constant or background not yet cached) breaks that, and the conv then waits for it to complete
    instead of polling the counters."""
    B, H, W, cin = x.shape
    taps = weight.shape[0]
    fills = _CONV2D_FILLS
    wp = conv2d_pack_cached(weight)
    d = Conv2dDesc()
    d.batch, d.H, d.W, d.cin, d.cin_stored = B, H, W, cin, x.planes.shape[-1]
    d.cout, d.taps, d.relu = cout, taps, 1 if relu else 0
    d.tile_order = CONV2D_TILE_ORDER
    d.n_split = 0        # the kernel picks its units (cout > 128: two 128-channel units per tile)
    d.out_ready = None if out_ready is None else _ptr(out_ready).value
    osp = of = None
    if out_split:
        cs = (cout + 63) // 64 * 64
        osp = torch.empty((2, B, H, W, cs), dtype=torch.float16, device=x.device)   # the kernel zeroes [cout, cs)
        d.out_split_ch = cs
    if out_f32:
        stride = (cout + 3) // 4 * 4
        of = torch.empty((B, H, W, stride), dtype=torch.float32, device=x.device)
        d.out_f32_stride = stride
    label = "conv2d_tma[taps=%d %d->%d]" % (taps, cin, cout)
    dist = x.tile_dist if TILE_OCCUPANCY else None
    reach, cvec, bg_sp, bg_f = 0, None, None, None
    if dist is not None:
        reach = x.reach + (1 if taps == 9 else 0)
        if not tile_skipping_valid(H, W, reach):
            dist = None        # the map is computed in full from here on (see tile_skipping_valid)
    if dist is not None:
        cvec = conv_constant(x.const, cin, weight, scale, shift, relu, cout)
        bg = conv_background(x, weight, scale, shift, relu, cout, out_split, out_f32)
        if bg is not None:
            bg_sp, bg_f = bg
    # with a cache filled above, the kernel would read what that work writes without waiting for it
    d.in_ready = None if in_ready is None or _CONV2D_FILLS != fills else _ptr(in_ready).value
    _call("sassd_conv2d_f16x3_occ_bg_status", label, ctypes.byref(d), _ptr(x.planes), _ptr(wp), _ptr(scale), _ptr(shift),
          _ptr(of), _ptr(osp), _ptr(dist), reach, _ptr(cvec), _ptr(bg_sp.planes if bg_sp is not None else None),
          _ptr(bg_f), _ptr(CONV2D_COUNTERS.get(label) if CONV2D_COUNTERS is not None else None), _ptr(x.status),
          _stream())
    return (SplitMap(osp, cout, dist, reach, cvec, bg_sp, x.status) if osp is not None else None), of


# ---------------------------------------------------------------------------- sparse conv on split rows
def features_to_split(feat, d_rows=None, status=None):
    """fp32 rows [cap, C] -> split rows [2, cap, cs] fp16 (cs = C rounded up to 8); F16_RANGE in ``status`` when a
    finite value has |x| >= 65520."""
    cap, C = feat.shape
    cs = (C + 7) // 8 * 8
    out = torch.empty((2, cap, cs), dtype=torch.float16, device=feat.device)
    _call("sassd_features_to_split_status", None, _ptr(feat), _ptr(d_rows), cap, C, cs, _ptr(out), _ptr(status), _stream())
    return out


def split_rows_float(planes, channels):
    """fp32 reconstruction of split rows (API-compat consumers and tests)."""
    return (planes[0].float() + planes[1].float() * (1.0 / 2048.0))[:, :channels].contiguous()


SPCONV_COUNTERS = None     # bench instrumentation: int32[2] device tensor -> += executed (tile, chunk) pairs, += tiles
SPCONV_TAP_SKIP = os.environ.get("SASSD_SPS_SKIP", "1") != "0"      # use the rulebook's tile masks
SPCONV_TAP_SPLIT = os.environ.get("SASSD_SPS_SPLIT", "1") != "0"    # chunk deal over all SMs for layers with few tiles
# Each tile walks its chunks from a tile-dependent chunk (spreads the weight reads over L2).  A row's summation order
# then depends on its tile's index, i.e. on the rows of the frames before it in the batch; False walks every tile from
# chunk 0, which makes each frame's bits independent of its batch (with SPCONV_TAP_SPLIT False too).
SPCONV_TAP_ROTATE = True


def spconv_split(planes, weight, scale, shift, relu, cout, rows_cap, nbr=None, d_rows=None, want_f32=False,
                 tile_mask=None, ws=None, status=None):
    """planes [2, in_cap, cin_stored] fp16; weight [taps, cin, cout] fp32 (packed on first use).
    Returns (out planes [2, rows_cap, out_ch], fp32 rows or None).  F16_RANGE in ``status`` when an output overflows
    the split."""
    taps = weight.shape[0]
    wp = spconv_pack_cached(weight, planes.shape[2])
    d = SpconvDesc()
    d.cin, d.cout, d.taps = planes.shape[2], cout, taps
    d.rows_cap, d.in_rows_cap, d.relu = rows_cap, planes.shape[1], 1 if relu else 0
    d.out_ch = (cout + 7) // 8 * 8
    d.fixed_walk = 0 if SPCONV_TAP_ROTATE else 1
    out = torch.empty((2, rows_cap, d.out_ch), dtype=torch.float16, device=planes.device)
    of = None
    if want_f32:
        d.out_f32_stride = (cout + 3) // 4 * 4
        of = torch.empty((rows_cap, d.out_f32_stride), dtype=torch.float32, device=planes.device)
    label = "spconv_split[taps=%d %d->%d]" % (taps, weight.shape[1], cout)
    w = None
    if SPCONV_TAP_SPLIT and taps > 1:
        w = (ws or _WS).get("spconv_split", _L().sassd_spconv_workspace_bytes(), planes.device, zeroed=True)
    _call("sassd_spconv_f16x3_status", label, ctypes.byref(d), _ptr(planes), _ptr(wp), _ptr(scale), _ptr(shift), _ptr(nbr),
          _ptr(tile_mask if SPCONV_TAP_SKIP else None), _ptr(d_rows), _ptr(out), _ptr(of), _ptr(w),
          0 if w is None else w.numel(), _ptr(SPCONV_COUNTERS), _ptr(status), _stream())
    return out, of


def split_rows_to_bev(planes, coors, d_rows, C, D, H, W, batch, status=None):
    bev = torch.zeros((2, batch, H, W, D * C), dtype=torch.float16, device=planes.device)
    dist = _tile_dist(batch, H, W, planes.device)
    _call("sassd_split_rows_to_bev", None, _ptr(planes), _ptr(coors), _ptr(d_rows), planes.shape[1], C, D, H, W, batch,
          _ptr(bev), _ptr(dist), _stream())
    return SplitMap(bev, D * C, dist, status=status)

"""ctypes binding of the C ABI declared in include/sassd_b200.h.

The CUDA library is the product: there is no CPU or eager fallback.  If
libsassd_b200.so is missing or a symbol is absent this module raises — loudly —
instead of degrading."""
import ctypes
import os

from . import build as _build

c_int, c_float, c_size_t, c_void_p = ctypes.c_int, ctypes.c_float, ctypes.c_size_t, ctypes.c_void_p


class VoxelParams(ctypes.Structure):
    _fields_ = [("voxel_size", c_float * 3), ("range_min", c_float * 3), ("grid", ctypes.c_int32 * 3),
                ("max_points", ctypes.c_int32), ("max_voxels", ctypes.c_int32)]


class Conv2dDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("batch", "H", "W", "cin", "cin_stored", "cout", "taps", "relu",
                                              "out_f32_stride", "out_split_ch", "tile_order", "n_split")] + \
               [("in_ready", c_void_p), ("out_ready", c_void_p)]


class SpconvDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("cin", "cout", "taps", "rows_cap", "in_rows_cap", "relu", "out_ch",
                                              "out_f32_stride", "fixed_walk")]


class GConvDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("mode", "precision", "cin", "cout", "taps", "in_stride", "out_stride",
                                              "rows_cap", "batch", "H", "W", "relu")]


class KittiEvalDesc(ctypes.Structure):
    _fields_ = ([(n, ctypes.c_int32) for n in ("nsets", "nframes", "nclass", "ndiff", "nover", "max_nd", "max_ng")]
                + [(n, c_void_p) for n in ("gt_off", "dt_off", "ov_off", "gt_dc", "gt_bbox", "dt_bbox", "dt_score",
                                           "ov_bbox", "ov_bev", "ov_3d", "aos_table", "compute_aos", "min_overlaps",
                                           "ign_gt", "ign_dt", "n_valid", "score_off")])


class PointLevels(ctypes.Structure):
    _fields_ = [("rows", c_void_p), ("plane_stride", ctypes.c_int64), ("row_stride", ctypes.c_int32),
                ("channels", ctypes.c_int32), ("split", ctypes.c_int32), ("pad", ctypes.c_int32)]


GCONV_TABLE, GCONV_CONV2D, GCONV_ROWS = 0, 1, 2
PREC_FP32, PREC_TF32X3, PREC_F16X3 = 0, 1, 2
CONV2D_TILE_H, CONV2D_TILE_W = 8, 16      # SASSD_CONV2D_TILE_H / _W of the header
TILE_DIST_MAX = 9                         # SASSD_TILE_DIST_MAX
SPCONV_TILE_ROWS = 128                    # SASSD_SPCONV_TILE_ROWS
KITTI_META, KITTI_ROW = 36, 14            # SASSD_KITTI_META / SASSD_KITTI_ROW
POINT_LEVEL_CHANNELS = (32, 64, 64)       # sassd_point_aux_head: features of backbone levels 1..3 (conv1, conv2, conv3)
POINT_FC_IN, POINT_FC_OUT = 160, 64       # point_fc: Linear(160, 64); point_cls / point_reg read its 64 outputs
KITTI_PARSE_DEFER, KITTI_PARSE_SCORE = 1, 2     # SASSD_KITTI_PARSE_DEFER / _SCORE: sassd_kitti_scan_labels' flags
GT_CAP_MAX = 256                          # SASSD_GT_CAP_MAX: ground-truth boxes per frame the loss kernels take
MERGE_MAX = 16                            # SASSD_MERGE_MAX: members sassd_merge_detections takes
# SASSD_KITTI_DT_*: a detection's state in the KITTI match table
KITTI_DT_NOT_COUNTED, KITTI_DT_TP, KITTI_DT_FP, KITTI_DT_DONTCARE, KITTI_DT_IGNORED = 0, 1, 2, 3, 4

OK = 0
ERRORS = {-1: "SASSD_ERR_ARG", -2: "SASSD_ERR_LAUNCH", -3: "SASSD_ERR_WORKSPACE", -4: "SASSD_ERR_UNSUPPORTED"}
FLAGS = {1: "VOXEL_CAP", 2: "ROWS_CAP", 4: "GUIDED_CAP", 8: "NMS_CAP", 16: "HASH_FULL", 32: "DET_CAP",
         64: "GT_CAP", 128: "GATHER_CAP", 256: "POINTS_CAP", 512: "F16_RANGE", 1024: "TILE_WAIT"}
F16_RANGE = 512                           # SASSD_FLAG_F16_RANGE: a finite value with |x| >= 65520 overflowed the fp16 split
F16_SPLIT_MAX = 65520.0                   # the least magnitude the 3xFP16 split cannot hold (half_rn rounds it to inf)
GATHER_CAP = 128                          # SASSD_FLAG_GATHER_CAP: sassd_points_in_rbboxes' rows exceed gather_cap
TILE_WAIT = 1024                          # SASSD_FLAG_TILE_WAIT: a dense conv gave up waiting for its input tiles

P = c_void_p
_SIGNATURES = {
    "sassd_version": (c_int, []),
    "sassd_voxelize_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "sassd_voxelize": (c_int, [P, P, c_int, c_int, ctypes.POINTER(VoxelParams), c_int, P, P, P, P, c_int, P, P, P,
                               c_size_t, P]),
    "sassd_voxel_mean": (c_int, [P, P, P, c_int, c_int, P, P]),
    "sassd_frustum_crop_workspace_bytes": (c_size_t, [c_int, c_int]),
    "sassd_frustum_crop": (c_int, [P, P, c_int, c_int, P, P, P, P, c_size_t, P]),
    "sassd_image_fov_crop": (c_int, [P, P, c_int, c_int, P, c_float, P, P, P, c_size_t, P]),
    "sassd_points_in_rbboxes_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "sassd_points_in_rbboxes": (c_int, [P, P, c_int, c_int, P, P, P, c_int, P, P, P, c_int, P, P, c_size_t, P]),
    "sassd_augment_drop_points": (c_int, [P, P, c_int, c_int, P, P, P, P, P, c_size_t, P]),
    "sassd_augment_noise_search": (c_int, [P, P, P, c_int, c_int, P, P, P, P, P]),
    "sassd_augment_assemble": (c_int, [P, P, c_int, P, P, c_int, P, P, P, P, P, P, P, P, c_int, P, P, P, c_int, P, P,
                                       P, P]),
    "sassd_anchor_mask_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "sassd_anchor_mask": (c_int, [P, P, c_int, c_int, c_int, c_int, P, c_int, c_int, P, P, c_size_t, P]),
    "sassd_hash_build": (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, P, P, c_int, P, P]),
    "sassd_rulebook_subm": (c_int, [P, P, c_int, c_int, c_int, c_int, P, P, c_int, P, P, P]),
    "sassd_rulebook_conv_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "sassd_rulebook_conv_outputs": (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, P, P, c_int, P, P, c_size_t, P]),
    "sassd_set_pdl": (c_int, [c_int]),
    "sassd_pdl_enabled": (c_int, []),
    "sassd_rulebook_conv_outputs_hash": (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, P, P, c_int, P, P, c_int, P, P,
                                                 c_size_t, P]),
    "sassd_rulebook_conv_nbr": (c_int, [P, P, c_int, c_int, c_int, c_int, P, P, c_int, P, P, P]),
    "sassd_rulebook_pairs": (c_int, [P, P, c_int, P, P, P]),
    "sassd_gconv": (c_int, [ctypes.POINTER(GConvDesc), P, P, P, P, P, P, P, P]),
    "sassd_gconv_status": (c_int, [ctypes.POINTER(GConvDesc), P, P, P, P, P, P, P, P, P]),
    "sassd_gconv_pack_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "sassd_gconv_pack": (c_int, [P, c_int, c_int, c_int, c_int, P, P]),
    "sassd_conv2d_pack_bytes": (c_size_t, [c_int, c_int, c_int]),
    "sassd_conv2d_pack": (c_int, [P, c_int, c_int, c_int, P, P]),
    "sassd_conv2d_f16x3": (c_int, [ctypes.POINTER(Conv2dDesc), P, P, P, P, P, P, P]),
    "sassd_conv2d_f16x3_occ": (c_int, [ctypes.POINTER(Conv2dDesc), P, P, P, P, P, P, P, c_int, P, P, P]),
    "sassd_conv2d_f16x3_occ_bg": (c_int, [ctypes.POINTER(Conv2dDesc), P, P, P, P, P, P, P, c_int, P, P, P, P, P]),
    "sassd_conv2d_f16x3_occ_bg_status": (c_int, [ctypes.POINTER(Conv2dDesc), P, P, P, P, P, P, P, c_int, P, P, P, P, P,
                                                 P]),
    "sassd_rotate_overlap_eval": (c_int, [P, P, P, P, P, c_int, c_int, c_int, P, P]),
    "sassd_kitti_match": (c_int, [c_int, P, P, P, P, P, P, P, P, P, P, P, P, c_int, ctypes.c_double, c_int, c_int, P, P,
                                  P, P]),
    "sassd_kitti_eval_flags": (c_int, [c_int, P, P, P, P, c_int, P, P, c_int, P, c_int, P, P, P, P, P]),
    "sassd_kitti_eval_flags_ranged": (c_int, [c_int, P, P, P, P, P, c_int, P, P, P, c_int, P, c_int, P, P, P, P, P,
                                              P, P, P]),
    "sassd_kitti_eval_overlaps": (c_int, [c_int, c_int, P, P, P, P, P, P, P, P, P, c_int, P, P, P, P]),
    "sassd_kitti_aos_table": (c_int, [c_int, c_int, P, P, P, P, P, P]),
    "sassd_kitti_eval_workspace_bytes": (c_size_t, [c_int, c_int]),
    "sassd_kitti_eval_match": (c_int, [ctypes.POINTER(KittiEvalDesc), P, P, P, P, P, P, c_size_t, P]),
    "sassd_kitti_eval_assign": (c_int, [ctypes.POINTER(KittiEvalDesc), c_int, c_int, P, P, P, P, P, P, P, c_size_t, P]),
    "sassd_kitti_boot_prepare": (c_int, [ctypes.POINTER(KittiEvalDesc), P, P, P, P, P, P, P, P, P, c_size_t, P]),
    "sassd_kitti_boot_eval": (c_int, [ctypes.POINTER(KittiEvalDesc), c_int] + [P] * 16),
    "sassd_kitti_assign": (c_int, [c_int, P, P, P, P, P, P, P, P, P, P, c_int, ctypes.c_double, P, P, P]),
    "sassd_kitti_scan_labels": (c_int, [P, P, c_int, P, P, P]),
    "sassd_kitti_parse_workspace_bytes": (c_size_t, [c_int]),
    "sassd_kitti_parse_labels": (c_int, [P, P, c_int, P, P, c_int, P, P, c_int, P, P, P, P, P, P, P, P, P, c_size_t, P]),
    "sassd_spconv_pack_bytes": (c_size_t, [c_int, c_int, c_int]),
    "sassd_spconv_pack": (c_int, [P, c_int, c_int, c_int, c_int, P, P]),
    "sassd_spconv_workspace_bytes": (c_size_t, []),
    "sassd_spconv_f16x3": (c_int, [ctypes.POINTER(SpconvDesc), P, P, P, P, P, P, P, P, P, P, c_size_t, P, P]),
    "sassd_spconv_f16x3_status": (c_int, [ctypes.POINTER(SpconvDesc), P, P, P, P, P, P, P, P, P, P, c_size_t, P, P, P]),
    "sassd_features_to_split": (c_int, [P, P, c_int, c_int, c_int, P, P]),
    "sassd_features_to_split_status": (c_int, [P, P, c_int, c_int, c_int, P, P, P]),
    "sassd_split_rows_to_bev": (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, P, P, P]),
    "sassd_sparse_to_bev_split": (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, P, P, P]),
    "sassd_sparse_to_bev_split_status": (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, P, P, P, P]),
    "sassd_sparse_to_bev": (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_int, P, P]),
    "sassd_decode_select_workspace_bytes": (c_size_t, [c_int, c_int]),
    "sassd_decode_select": (c_int, [P, c_int, c_int, c_int, c_int, c_int, P, c_int, P, c_int, c_float, P, P, P, P, c_int, P,
                                    P, c_size_t, P]),
    "sassd_pswarp": (c_int, [P, c_int, c_int, c_int, c_int, P, P, c_int, c_float, c_float, c_float, P, P]),
    "sassd_rescore_nms_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "sassd_rescore_nms": (c_int, [P, P, P, P, c_int, c_int, c_float, c_float, c_int, P, P, c_int, P, P, c_size_t, P]),
    "sassd_kitti_format": (c_int, [P, P, c_int, c_int, P, P, P, P]),
    "sassd_merge_detections": (c_int, [P, P, P, P, c_int, c_int, P, P, P]),
    "sassd_three_nn": (c_int, [P, P, P, c_int, P, P, P, P, P, P, P, P, P, P]),
    "sassd_point_aux_head": (c_int, [P, P, P, c_int, ctypes.POINTER(PointLevels), P, P, P, P, P]),
    "sassd_nms_workspace_bytes": (c_size_t, [c_int]),
    "sassd_nms_mask": (c_int, [P, c_int, c_float, P, P]),
    "sassd_nms_sorted": (c_int, [P, c_int, c_float, P, P, P, c_size_t, P]),
    "sassd_boxes_iou_bev": (c_int, [P, c_int, P, c_int, P, P]),
    "sassd_loss_workspace_bytes": (c_size_t, [c_int, c_int]),
    "sassd_points_in_boxes": (c_int, [P, P, c_int, P, P, c_int, c_int, P, P, P, P, P]),
    "sassd_assign_rpn": (c_int, [P, c_int, P, c_int, c_int, P, P, P, P, c_int, c_int, P, P, P, P, P, P, P, P, c_size_t,
                                 P]),
    "sassd_assign_pswarp": (c_int, [P, P, c_int, c_int, P, c_int, P, c_int, P, c_float, c_float, P, P, P, P, P, c_size_t,
                                    P]),
    "sassd_rpn_loss": (c_int, [P, c_int, c_int, c_int, c_int, c_int, P, c_int, c_int, P, P, P, P, P, c_size_t, P]),
    "sassd_pswarp_loss": (c_int, [P, P, c_int, c_int, P, P, P, c_size_t, P]),
    "sassd_aux_loss": (c_int, [P, P, P, P, P, c_int, c_int, P, P, P, c_size_t, P]),
}

_LIB = None


class SassdError(RuntimeError):
    pass


def exported_symbols():
    return sorted(_SIGNATURES)


def load(build_if_missing=True):
    """Load libsassd_b200.so and bind every symbol of include/sassd_b200.h."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = _build.LIB
    if not os.path.exists(path):
        if not build_if_missing:
            raise SassdError("libsassd_b200.so not built: run `python -m sassd_b200.build`")
        path = _build.build()
    lib = ctypes.CDLL(path)
    for name, (res, args) in _SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise SassdError("libsassd_b200.so lacks symbol %s (stale build?)" % name) from e
        fn.restype = res
        fn.argtypes = args
    _LIB = lib
    return lib


def check(rc, what):
    if rc != OK:
        raise SassdError("%s failed: %s (%d)" % (what, ERRORS.get(rc, "unknown"), rc))


def decode_flags(word):
    return [name for bit, name in FLAGS.items() if word & bit]


def raise_on_status(word):
    """Raise SassdError naming the capacities that overflowed if the status word ``d_status`` of a step has a
    SASSD_FLAG_* bit set.  ``word`` is an int or a one-element tensor (a device tensor is read with a sync)."""
    word = int(word)
    if word & F16_RANGE:
        raise SassdError("activation out of the fp16 split's range on device (|x| >= 65520), outputs that read it are "
                         "NaN: %s; run the model at set_precision(PREC_FP32) (fp32 range)" % decode_flags(word))
    if word & TILE_WAIT:
        raise SassdError("a dense conv waited over a second for its input tiles and went on without them, its outputs "
                         "are undefined: %s; SASSD_TILE_FLAGS=0 turns the per-tile waits off" % decode_flags(word))
    if word:
        raise SassdError("capacity overflow on device: %s" % decode_flags(word))

/* sassd_b200 — C ABI of the SA-SSD inference hot path for the H100 (sm_90a).
 *
 * Drop-in boundary (DESIGN.md §Boundary, SURVEY.md §8b): these are the entry
 * points a binding of the reference's native extensions for this path would
 * call.  Plain C: device pointers, sizes, a CUDA stream; no torch types.
 *
 * Conventions (differences from the reference ABI are deliberate and listed):
 *  - every pointer is a DEVICE pointer unless the name says host_;
 *  - every function takes the stream to launch on (the reference launches on
 *    the legacy default stream, iou3d_kernel.cu:359-386) and returns an int
 *    status (SASSD_OK or a negative SASSD_ERR_*); nothing exits the process
 *    (the reference calls exit(), iou3d.cpp:13-21) and nothing is allocated or
 *    freed inside a call (the reference cudaMalloc/cudaFree's per NMS call,
 *    iou3d.cpp:87,98) — scratch comes in through `ws` with a *_workspace_bytes query;
 *  - data-dependent sizes (voxel counts, active rows, guided anchors, kept boxes)
 *    live in device memory (`d_*` int32 counters) so that a whole frame runs
 *    without a host round trip and can be captured in a CUDA graph; buffers are
 *    sized by capacity (`*_cap`).  A capacity overflow truncates the output and
 *    sets a bit in the int32 word `d_status` (SASSD_FLAG_*).
 *  - layouts: points [N,4] f32 (x,y,z,r); voxel coordinates int32 (b,z,y,x);
 *    boxes [x,y,z(bottom),w,l,h,ry]; BEV boxes [x1,y1,x2,y2,ry];
 *    feature matrices row-major [rows, channels]; dense maps NHWC.
 */
#ifndef SASSD_B200_H
#define SASSD_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* sassd_stream_t; /* cudaStream_t */

enum {
    SASSD_OK = 0,
    SASSD_ERR_ARG = -1,       /* bad argument (null pointer, unsupported size) */
    SASSD_ERR_LAUNCH = -2,    /* CUDA reported a launch error */
    SASSD_ERR_WORKSPACE = -3, /* workspace too small */
    SASSD_ERR_UNSUPPORTED = -4
};

enum { /* bits of *d_status */
    SASSD_FLAG_VOXEL_CAP = 1,   /* more voxel rows than the output capacity */
    SASSD_FLAG_ROWS_CAP = 2,    /* strided-conv output rows exceed capacity */
    SASSD_FLAG_GUIDED_CAP = 4,  /* guided anchors per frame exceed capacity: the first k_cap selected anchors in
                                   anchor order are kept (sassd_decode_select) */
    SASSD_FLAG_NMS_CAP = 8,     /* NMS candidates per frame exceed capacity: the NMS runs on the first 4096 score
                                   passers in candidate order (sassd_rescore_nms) */
    SASSD_FLAG_HASH_FULL = 16,
    SASSD_FLAG_DET_CAP = 32,    /* boxes kept by the NMS exceed the detection capacity: the first det_cap kept
                                   boxes in score order are returned */
    SASSD_FLAG_GT_CAP = 64,     /* ground-truth boxes per frame exceed gt_cap: the first gt_cap boxes are used
                                   (sassd_points_in_boxes, sassd_assign_*, sassd_points_in_rbboxes) */
    SASSD_FLAG_GATHER_CAP = 128, /* gathered rows exceed gather_cap: rows past it are not written
                                   (sassd_points_in_rbboxes) */
    SASSD_FLAG_POINTS_CAP = 256, /* augmented rows exceed out_cap: rows past it are not written
                                   (sassd_augment_assemble) */
    SASSD_FLAG_TILE_WAIT = 1024, /* a dense conv waited longer than about a second for its input tiles' ready counters
                                   (sassd_conv2d_desc.in_ready) and went on without them: its outputs are undefined */
    SASSD_FLAG_F16_RANGE = 512  /* a finite value at or above 65520 in magnitude was split into fp16 planes: its hi half is
                                   +-inf and its lo half -+inf, so every output that reads it becomes NaN.  Set by the
                                   split stores of the *_status entry points (sassd_conv2d_f16x3_occ_bg_status,
                                   sassd_spconv_f16x3_status, sassd_features_to_split_status,
                                   sassd_sparse_to_bev_split_status, and sassd_gconv_status's on-the-fly input split at
                                   SASSD_PREC_F16X3); values that are already inf or NaN do not set it.  The FP32 and
                                   TF32X3 precisions have fp32's range */
};

int sassd_version(void);
/* Launch hint, process-wide: on != 0 launches the tensor-core conv kernels as programmatic dependents of their
 * predecessors (their prologues overlap the previous layer's tail); -1 restores the default (environment SASSD_PDL,
 * else off).  Worth ~2 % for a step that runs alone on the GPU, costs throughput when several steps are in flight, so set
 * it around the capture of a latency-oriented graph only.  Returns the previous setting.  Results never change. */
int sassd_set_pdl(int on);
/* Whether launches are programmatic dependents now (sassd_set_pdl, else the environment). */
int sassd_pdl_enabled(void);

/* ------------------------------------------------------------------------
 * Voxelization.  Replaces mmdet/ops/points_op/points_ops.py:104-164
 * (points_to_voxel, reverse_index=True) called from
 * mmdet/core/point_cloud/voxel_generator.py:22-25, fused with
 * SingleStageDetector.merge_second_batch's batch-index padding
 * (mmdet/models/detectors/single_stage.py:57-65) and SimpleVoxel.forward
 * (mmdet/models/backbones/vxnet.py:110-116).
 *
 * points: frames concatenated, frame b = rows [pt_off[b], pt_off[b+1]).
 * Outputs are bit-identical to the sequential reference per frame (first-touch
 * voxel order, first `max_points` points, stop at voxel `max_voxels`), rows of
 * frame b start at sum of the previous frames' counts:
 *   voxels [rows_cap, max_points, 4] (zero padded), coors [rows_cap,4] (b,z,y,x),
 *   num_points [rows_cap], mean [rows_cap,4] (may be NULL),
 *   d_frame_rows [batch+1] = exclusive row offsets, last = total rows.
 * ---------------------------------------------------------------------- */
typedef struct {
    float voxel_size[3];  /* x, y, z */
    float range_min[3];   /* x, y, z */
    int32_t grid[3];      /* x, y, z cells (1408, 1600, 40 under car_cfg) */
    int32_t max_points;   /* <= 8 */
    int32_t max_voxels;
} sassd_voxel_params;

size_t sassd_voxelize_workspace_bytes(int n_points_cap, int batch, int slots_per_frame);
int sassd_voxelize(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch,
                   const sassd_voxel_params* host_params, int slots_per_frame,
                   float* voxels, int32_t* coors, int32_t* num_points, float* mean, int rows_cap,
                   int32_t* d_frame_rows, int32_t* d_status, void* ws, size_t ws_bytes, sassd_stream_t stream);

/* SimpleVoxel.forward alone (vxnet.py:110-116): mean[r,:] = sum_s voxels[r,s,:4] / num_points[r]. */
int sassd_voxel_mean(const float* voxels, const int32_t* num_points, const int32_t* d_rows, int rows_cap,
                     int max_points, float* mean, sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * Camera-frustum crop of full sweeps.  Replaces the offline reduced-cloud
 * step, tools/create_data.py:107-140 -> remove_outside_points
 * (mmdet/core/bbox3d/geometry.py:50-61), on the device.
 *
 * points [n_points_cap,4], frame b = rows [d_pt_off[b], d_pt_off[b+1]) as for
 * sassd_voxelize; planes [batch][6][4] fp64 (n.x, n.y, n.z, d per face, the
 * normals pointing into the frustum).  Point i of frame b is kept when
 * s = ((x*n.x + y*n.y) + z*n.z) + d is < 0 for all 6 faces, evaluated in fp64
 * in that order without contraction (points_in_convex_polygon_3d_jit,
 * geometry.py:190-222: `s >= 0` rejects, so a NaN coordinate keeps the point).
 * Kept rows are compacted in input order, frames concatenated:
 * points_out [n_points_cap,4], d_pt_off_out [batch+1].  One pass, no host
 * synchronisation: graph-capturable.  batch <= 256.
 * ---------------------------------------------------------------------- */
size_t sassd_frustum_crop_workspace_bytes(int n_points_cap, int batch);
int sassd_frustum_crop(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch,
                       const double* planes, float* points_out, int32_t* d_pt_off_out,
                       void* ws, size_t ws_bytes, sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * Image-FOV crop of full sweeps: the reference's raw-drive dataset
 * (KittiVideo, mmdet/datasets/kitti.py:394) crops every sweep with
 * get_lidar_in_image_fov(points, calib, 0, 0, w, h, clip_distance=0.1)
 * (mmdet/datasets/kitti_utils.py:252-263).
 *
 * points / d_pt_off as for sassd_frustum_crop; meta [batch][SASSD_KITTI_META]
 * fp64 is the per-frame block of sassd_kitti_format (P2, Tr_velo_to_cam,
 * R0_rect, img_h, img_w).  Per point, in fp64 from the widened x, y, z:
 * ref = [x,y,z,1] V2C^T, rect = ref R0^T, uvw = [rect,1] P2^T, every dot
 * product a sequential FMA chain from k = 0; u = uvw0/uvw2, v = uvw1/uvw2
 * (IEEE division).  Kept when u < img_w && u >= 0 && v < img_h && v >= 0
 * && x > clip_x (fp32 comparison); a NaN coordinate drops the point.
 * Compaction, outputs, workspace (sassd_frustum_crop_workspace_bytes),
 * argument checks and error codes are those of sassd_frustum_crop.
 * ---------------------------------------------------------------------- */
int sassd_image_fov_crop(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch,
                         const double* meta, float clip_x, float* points_out, int32_t* d_pt_off_out,
                         void* ws, size_t ws_bytes, sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * Points in rotated boxes, gathered per box: the reference's ground-truth
 * database and num_points_in_gt (tools/create_data.py:16-45, 233-240 ->
 * points_in_rbbox, mmdet/core/bbox3d/geometry.py:63-74, 190-226).
 *
 * points / d_pt_off as for sassd_frustum_crop (the cropped frames);
 * planes [batch][box_cap][6][4] fp64 (n.x, n.y, n.z, d, inward normals),
 * centres [batch][box_cap][3] fp64 (box x, y, z, LiDAR frame), d_nbox [batch]:
 * slots j < d_nbox[b] of frame b are boxes.  Point i of frame b is in box j
 * under sassd_frustum_crop's test (fp64, no contraction, `s >= 0` rejects:
 * a NaN coordinate is in every box, a box of zero size holds nothing); a point
 * may be in several boxes.  Outputs:
 *   counts [batch][box_cap]       members per slot (0 for empty slots),
 *   seg_off [batch*box_cap + 1]   exclusive offsets of the slots' rows,
 *   gathered [gather_cap][4]      box (b, j)'s members in input order, each
 *                                 x, y, z as (float)((double)p - centre) and
 *                                 the reflectance unchanged (a NaN keeps its bits).
 * More rows than gather_cap: the rest are not written and
 * SASSD_FLAG_GATHER_CAP is set (counts and seg_off stay exact); d_nbox[b] >
 * box_cap sets SASSD_FLAG_GT_CAP and uses the first box_cap boxes.  gathered
 * may be NULL when gather_cap is 0 (counts only).  box_cap <= SASSD_GT_CAP_MAX,
 * batch <= 256.  No host synchronisation, no allocation: graph-capturable.
 * Argument checks and error codes as for sassd_frustum_crop.
 * ---------------------------------------------------------------------- */
size_t sassd_points_in_rbboxes_workspace_bytes(int n_points_cap, int batch, int box_cap);
int sassd_points_in_rbboxes(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch,
                            const double* planes, const double* centres, const int32_t* d_nbox, int box_cap,
                            int32_t* counts, int32_t* seg_off, float* gathered, int gather_cap,
                            int32_t* d_status, void* ws, size_t ws_bytes, sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * anchors_mask.  Replaces mmdet/datasets/kitti.py:333-343 +
 * mmdet/core/bbox3d/geometry.py:675-709 (occupancy count, two cumsums,
 * integral-image lookup, `> threshold`).  rects [n_anchors,4] int32 are the
 * clamped cell indices (c0,c1,c2,c3) of each anchor's near-axis-aligned
 * footprint — static, computed once on the host with the reference's fp32
 * arithmetic.  mask [batch, n_anchors] uint8.
 * ---------------------------------------------------------------------- */
size_t sassd_anchor_mask_workspace_bytes(int batch, int H, int W);
int sassd_anchor_mask(const int32_t* coors, const int32_t* d_rows, int rows_cap, int batch, int H, int W,
                      const int32_t* rects, int n_anchors, int threshold, uint8_t* mask,
                      void* ws, size_t ws_bytes, sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * Rulebooks.  Replace spconv v1.0 `get_indice_pairs` (third-party; call sites
 * mmdet/models/necks/cmn.py:139-173,197-212).  The hot path uses a neighbour
 * table nbr[n_out, 27] (input row feeding output row o through kernel offset
 * k = (kz*3+ky)*3+kx, -1 = none); sassd_rulebook_pairs re-indexes it into the
 * spconv-v1 tables indice_pairs[2,27,n_cap] / indice_pair_num[27] (canonical
 * order: per offset ascending output row).
 * ---------------------------------------------------------------------- */
/* hash index over active coordinates: keys/vals [slots] int32, slots a power of two >= 2*n_cap. */
int sassd_hash_build(const int32_t* coors, const int32_t* d_rows, int rows_cap, int batch, int D, int H, int W,
                     int32_t* keys, int32_t* vals, int slots, int32_t* d_status, sassd_stream_t stream);
/* submanifold 3x3x3: output sites == input sites. */
/* tile_mask (optional): int32 [ceil(rows_cap / 128)], bit k of entry t = some row of rows [128t, 128t+128) has a
 * neighbour at offset k (consumed by sassd_spconv_f16x3 to skip absent taps). */
int sassd_rulebook_subm(const int32_t* coors, const int32_t* d_rows, int rows_cap, int D, int H, int W,
                        const int32_t* keys, const int32_t* vals, int slots, int32_t* nbr, int32_t* tile_mask,
                        sassd_stream_t stream);
/* strided conv (k=3,s=2,p=1): active output set, sorted by flattened (b,z,y,x). */
size_t sassd_rulebook_conv_workspace_bytes(int batch, int Do, int Ho, int Wo);
int sassd_rulebook_conv_outputs(const int32_t* coors_in, const int32_t* d_rows_in, int rows_cap_in, int batch,
                                int D, int H, int W, int32_t* coors_out, int32_t* d_rows_out, int rows_cap_out,
                                int32_t* d_status, void* ws, size_t ws_bytes, sassd_stream_t stream);
/* Same, and every output row is inserted into the hash index of the OUTPUT level as it is written (keys_out / vals_out
 * [slots_out], slots_out a power of two >= 2 * rows_cap_out; cleared here), which replaces that level's
 * sassd_hash_build launch.  Two kernels: mark (bitmap over the output grid) and a single-pass compaction (block scan
 * + decoupled look-back over the chunks of the bitmap). */
int sassd_rulebook_conv_outputs_hash(const int32_t* coors_in, const int32_t* d_rows_in, int rows_cap_in, int batch,
                                     int D, int H, int W, int32_t* coors_out, int32_t* d_rows_out, int rows_cap_out,
                                     int32_t* keys_out, int32_t* vals_out, int slots_out, int32_t* d_status, void* ws,
                                     size_t ws_bytes, sassd_stream_t stream);
/* neighbour table of the strided conv: nbr[o][k] = row of input cell 2*o - 1 + k. */
int sassd_rulebook_conv_nbr(const int32_t* coors_out, const int32_t* d_rows_out, int rows_cap_out, int D, int H, int W,
                            const int32_t* keys_in, const int32_t* vals_in, int slots_in, int32_t* nbr,
                            int32_t* tile_mask, sassd_stream_t stream);
int sassd_rulebook_pairs(const int32_t* nbr, const int32_t* d_rows_out, int rows_cap, int32_t* indice_pairs,
                         int32_t* indice_pair_num, sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * Gathered implicit-GEMM convolution — one kernel family for
 *   SubMConv3d / SparseConv3d  (spconv v1.0 indice_conv; cmn.py:145-173,192-231)
 *   SparseConv3d 1x1x1         (cmn.py:208-212)
 *   nn.Conv2d 3x3 / 1x1 + BatchNorm2d(eval) + ReLU (BEVNet cmn.py:233-282,
 *     SSDRotateHead ssd_rotate_head.py:120-125,218-231, PSWarpHead.convs :424-429)
 *   out[m, :] = act( (sum_t in[row(m,t), :] @ W[t]) * scale + shift )
 * mode TABLE : row(m,t) = nbr[m*taps + t]            (sparse layers)
 * mode CONV2D: rows are pixels of a [batch,H,W] NHWC map, taps = 3x3 window, zero padding
 * mode ROWS  : taps == 1, row(m,0) = m                (1x1 convs / plain GEMM)
 * weight [taps, Cin, Cout] f32; scale/shift [Cout] (folded BatchNorm or bias); Cin % 4 == 0.
 * precision: SASSD_PREC_FP32 = CUDA-core FFMA; SASSD_PREC_TF32X3 / SASSD_PREC_F16X3 = Hopper tensor cores (wgmma) with a
 * 3-product hi/lo split of both operands (tf32: 21 bits, any range; fp16: 22 bits, |x| < 65520, 2x the MMA rate).
 * With relu a NaN output stays NaN (as torch.relu).
 * ---------------------------------------------------------------------- */
enum { SASSD_GCONV_TABLE = 0, SASSD_GCONV_CONV2D = 1, SASSD_GCONV_ROWS = 2 };
enum { SASSD_PREC_FP32 = 0, SASSD_PREC_TF32X3 = 1, SASSD_PREC_F16X3 = 2 };
typedef struct {
    int32_t mode, precision;
    int32_t cin, cout, taps;
    int32_t in_stride, out_stride; /* floats per row */
    int32_t rows_cap;              /* upper bound of rows (grid sizing) */
    int32_t batch, H, W;           /* CONV2D only */
    int32_t relu;
} sassd_gconv_desc;
int sassd_gconv(const sassd_gconv_desc* host_desc, const float* in, const float* weight, const float* scale,
                const float* shift, const int32_t* nbr, const int32_t* d_rows, float* out, sassd_stream_t stream);
/* Same, with a status word (nullable): SASSD_PREC_F16X3 sets SASSD_FLAG_F16_RANGE in it when an input value overflows
 * the split. */
int sassd_gconv_status(const sassd_gconv_desc* host_desc, const float* in, const float* weight, const float* scale,
                       const float* shift, const int32_t* nbr, const int32_t* d_rows, float* out, int32_t* d_status,
                       sassd_stream_t stream);

/* The tensor-core precisions take their weights pre-split (hi / lo) and pre-swizzled for the shared-memory
 * operand layout: pack once per layer with sassd_gconv_pack (weight [taps,cin,cout] fp32 -> packed,
 * sassd_gconv_pack_bytes bytes) and pass `packed` as `weight`. */
size_t sassd_gconv_pack_bytes(int taps, int cin, int cout, int precision);
int sassd_gconv_pack(const float* weight, int taps, int cin, int cout, int precision, void* packed,
                     sassd_stream_t stream);

/* Dense NHWC conv (3x3 pad 1, or 1x1) + folded BatchNorm + ReLU on the "split map" activation format — the
 * BEVNet / head convolutions (cmn.py:264-282, ssd_rotate_head.py:218-231,424-429) with the activation operand
 * moved by TMA (cp.async.bulk.tensor) instead of producer warps.  A split map is two fp16 planes
 * [2][batch][H][W][C] (C % 64 == 0): hi = half(x), lo = half((x - hi) * 2048).  Outputs: fp32 NHWC
 * (out_f32, stride out_f32_stride) and/or the next layer's split map (out_split, out_split_ch channels, the
 * channels beyond cout written as zero).  wpack: sassd_conv2d_pack.  16 < cout <= 256.  With relu a NaN output stays
 * NaN (as torch.relu). */
/* The weight pack of sassd_conv2d_f16x3*: weight [taps,cin,cout] fp32 -> packed (sassd_conv2d_pack_bytes bytes, 0 for
 * an unsupported shape).  cout <= 64: the SASSD_PREC_F16X3 pack of sassd_gconv_pack; cout > 64: the hi / lo fp16
 * weights in the register-fragment order of the kernel's wgmma A operand.  taps 9 or 1. */
size_t sassd_conv2d_pack_bytes(int taps, int cin, int cout);
int sassd_conv2d_pack(const float* weight, int taps, int cin, int cout, void* packed, sassd_stream_t stream);
typedef struct {
    int32_t batch, H, W;
    int32_t cin, cin_stored;       /* valid / stored input channels */
    int32_t cout, taps, relu;
    int32_t out_f32_stride, out_split_ch;
    int32_t tile_order;            /* sassd_conv2d_f16x3_occ: 0 = tiles round-robin over the CTAs (best with several steps
                                      in flight), 1 = computed tiles first, constant tiles after (best for one step at a
                                      time: no CTA gets two computed tiles while others only store constants); honoured
                                      for maps of up to 4608 tiles (16 frames of 200 x 176), round-robin above */
    int32_t n_split;               /* accepted for ABI compatibility and ignored: a work unit is a tile and at most 128 of
                                      its output channels (the register accumulators' budget), so cout > 128 always runs
                                      as two units per tile */
    /* Tile ready counters (NULL: off; only for cout > 64 with out_split_ch at most the units' 128 or 256 channels),
     * int32 [batch * tiles_y * tiles_x + 1] over the SASSD_CONV2D_TILE_H x SASSD_CONV2D_TILE_W tiles, zeroed before
     * the chain of launches that uses them and never reset by a kernel.  out_ready: this launch adds to a tile's
     * counter as its units store it, and to the last word once per CTA past its prologue.  in_ready: the out_ready of
     * the launch that wrote in_split, which must be the previous launch on the stream (anything launched in between
     * may still be running when this one reads what it wrote).  This launch then does not wait for that one to
     * complete before it starts, but loads each tile's inputs once the tiles they read are stored, and completes only
     * after it (results are the same bit for bit).  Needs d_status: a wait longer than about a second (a bug) stops
     * waiting and sets SASSD_FLAG_TILE_WAIT. */
    const int32_t* in_ready;
    int32_t* out_ready;
} sassd_conv2d_desc;
int sassd_conv2d_f16x3(const sassd_conv2d_desc* host_desc, const void* in_split, const void* wpack, const float* scale,
                       const float* shift, float* out_f32, void* out_split, sassd_stream_t stream);
/* Same, for maps that descend from a scattered sparse tensor and are therefore constant over large regions.
 * tile_dist[(b * tiles_y + ty) * tiles_x + tx] (written by sassd_split_rows_to_bev / sassd_sparse_to_bev_split into a
 * buffer pre-filled with a large value) is the Chebyshev distance in pixels from the SASSD_CONV2D_TILE_H x
 * SASSD_CONV2D_TILE_W tile to the nearest active cell of the scattered map.  `reach` = number of 3x3 convolutions
 * between that map and this layer's OUTPUT (1 for the first conv): a tile with tile_dist > reach that does not lie on
 * the image border (border tiles are always computed once reach >= 2, because the zero padding differs from the
 * constant) sees a constant input, so its output is the constant vector `const_out[cout]` (the caller obtains it by
 * running this same function on a small constant map - bit-identical to computing the tile).  Such tiles skip loads
 * and MMAs and only store.  tile_dist == NULL: plain sassd_conv2d_f16x3. */
#define SASSD_CONV2D_TILE_H 8
#define SASSD_CONV2D_TILE_W 16
#define SASSD_TILE_DIST_MAX 9          /* distances beyond this are stored as any larger value */
int sassd_conv2d_f16x3_occ(const sassd_conv2d_desc* host_desc, const void* in_split, const void* wpack,
                           const float* scale, const float* shift, float* out_f32, void* out_split,
                           const int32_t* tile_dist, int reach, const float* const_out, int32_t* counters,
                           sassd_stream_t stream);     /* counters: optional int32[2], += tiles computed, += tiles */
/* Same, with a background for the border tiles.  A tile on the image border with tile_dist > reach (reach >= 2) sees
 * only inactive cells and the zero padding, so its output does not depend on the frame: it equals, bit for bit, this
 * function's output on an empty scene at the same pixels (one output element per lane, a fixed chunk order, no
 * atomics).  bg_split [2][1][H][W][out_split_ch] / bg_f32 [1][H][W][out_f32_stride] hold that output - the layer run
 * with batch 1 and no tile skipping on the previous layer's background (an all-zero map for the first conv) - and
 * every frame's far border tiles copy it with 16-byte loads and stores, without loads of the input or MMAs.  Interior
 * far tiles still store const_out.  The background must hold every output the call writes (SASSD_ERR_ARG
 * otherwise); both NULL: sassd_conv2d_f16x3_occ, which computes the border tiles.  counters count computed tiles
 * only. */
int sassd_conv2d_f16x3_occ_bg(const sassd_conv2d_desc* host_desc, const void* in_split, const void* wpack,
                              const float* scale, const float* shift, float* out_f32, void* out_split,
                              const int32_t* tile_dist, int reach, const float* const_out, const void* bg_split,
                              const float* bg_f32, int32_t* counters, sassd_stream_t stream);
/* Same, with a status word (nullable; the three entry points above pass NULL): SASSD_FLAG_F16_RANGE is set when an
 * output stored into out_split overflows the split (|x| >= 65520). */
int sassd_conv2d_f16x3_occ_bg_status(const sassd_conv2d_desc* host_desc, const void* in_split, const void* wpack,
                                     const float* scale, const float* shift, float* out_f32, void* out_split,
                                     const int32_t* tile_dist, int reach, const float* const_out, const void* bg_split,
                                     const float* bg_f32, int32_t* counters, int32_t* d_status, sassd_stream_t stream);
/* dense() of the last sparse tensor straight into a (pre-zeroed) split map [2,batch,H,W,D*C]. */
int sassd_sparse_to_bev_split(const float* feat, const int32_t* coors, const int32_t* d_rows, int rows_cap, int C,
                              int D, int H, int W, int batch, void* bev_split, int32_t* tile_dist,
                              sassd_stream_t stream);   /* tile_dist: optional, pre-filled with a large value, see above */
/* Same, with a status word (nullable): SASSD_FLAG_F16_RANGE when a finite input has |x| >= 65520. */
int sassd_sparse_to_bev_split_status(const float* feat, const int32_t* coors, const int32_t* d_rows, int rows_cap,
                                     int C, int D, int H, int W, int batch, void* bev_split, int32_t* tile_dist,
                                     int32_t* d_status, sassd_stream_t stream);

/* Ruled sparse conv on "split rows" (two fp16 planes [2][rows][C], C % 8 == 0; hi = half(x), lo = half((x-hi)*2048)):
 * same semantics as sassd_gconv TABLE / ROWS mode with SASSD_PREC_F16X3, but the gather is 16-byte cp.async copies
 * straight into the tensor-core operand tiles and the epilogue writes the next layer's planes (out_split, out_ch
 * channels, zero beyond cout) and/or fp32 rows.  taps == 1: row(m) = m.  cin <= 64, cout <= 64. */
typedef struct {
    int32_t cin, cout, taps;         /* cin = stored channels of the input planes */
    int32_t rows_cap, in_rows_cap;   /* output rows capacity; rows of the input planes (plane stride) */
    int32_t relu, out_ch, out_f32_stride;
    int32_t fixed_walk;              /* 1: every tile walks its K chunks from chunk 0; 0 (default): from a tile-dependent
                                        chunk, which spreads the CTAs' weight reads over L2 but makes a row's fp32
                                        summation order depend on the index of its tile, i.e. on the rows before it */
} sassd_spconv_desc;
/* wpack for sassd_spconv_f16x3: weight [taps, cin, cout] fp32 -> sassd_spconv_pack_bytes(taps, cin_stored, cout)
 * bytes.  Narrow inputs are tap-packed: a 64-wide K chunk holds 64 / cin_stored taps (cin_stored 8, 16, 32). */
size_t sassd_spconv_pack_bytes(int taps, int cin_stored, int cout);
int sassd_spconv_pack(const float* weight, int taps, int cin, int cin_stored, int cout, void* packed,
                      sassd_stream_t stream);
/* tile_mask (optional, taps <= 27): int32 per SASSD_SPCONV_TILE_ROWS-row tile of the OUTPUT rows, bit t set when some
 * row of the tile has a neighbour at tap t (written by sassd_rulebook_subm / sassd_rulebook_conv_nbr); K chunks whose
 * taps are all absent are skipped (an absent pair contributes exactly zero, so the result is unchanged).
 * ws (optional, sassd_spconv_workspace_bytes(), zero-filled before its first use, not shared by calls that may run at
 * the same time): with it, a layer that has at most as many tiles as CTAs, and whose longest tile would otherwise
 * dominate, deals its tiles' active K chunks evenly over all CTAs; the fp32 partial sums of tiles cut between CTAs and the counters that pick the CTA finishing each tile live
 * in it, and every call leaves the counters zero again.  Without it, one CTA per tile.
 * counters (optional, int32[2], caller-zeroed): += executed (tile, chunk) pairs, += tiles (instrumentation).
 * With relu a NaN output stays NaN (as torch.relu); the columns >= cout are written as exact zeros whatever the inputs
 * hold. */
#define SASSD_SPCONV_TILE_ROWS 128
size_t sassd_spconv_workspace_bytes(void);
int sassd_spconv_f16x3(const sassd_spconv_desc* host_desc, const void* in_split, const void* wpack, const float* scale,
                       const float* shift, const int32_t* nbr, const int32_t* tile_mask, const int32_t* d_rows,
                       void* out_split, float* out_f32, void* ws, size_t ws_bytes, int32_t* counters,
                       sassd_stream_t stream);
/* Same, with a status word (nullable): SASSD_FLAG_F16_RANGE when an output stored into out_split overflows the split. */
int sassd_spconv_f16x3_status(const sassd_spconv_desc* host_desc, const void* in_split, const void* wpack,
                              const float* scale, const float* shift, const int32_t* nbr, const int32_t* tile_mask,
                              const int32_t* d_rows, void* out_split, float* out_f32, void* ws, size_t ws_bytes,
                              int32_t* counters, int32_t* d_status, sassd_stream_t stream);
/* fp32 rows [rows, cin] -> split rows [2][rows_cap][cs] (cs >= cin, cs % 8 == 0, padding zero). */
int sassd_features_to_split(const float* feat, const int32_t* d_rows, int rows_cap, int cin, int cs, void* out_split,
                            sassd_stream_t stream);
/* Same, with a status word (nullable): SASSD_FLAG_F16_RANGE when a finite input has |x| >= 65520. */
int sassd_features_to_split_status(const float* feat, const int32_t* d_rows, int rows_cap, int cin, int cs,
                                   void* out_split, int32_t* d_status, sassd_stream_t stream);
/* dense() of split rows into a (pre-zeroed) split BEV map [2,batch,H,W,D*C]. */
int sassd_split_rows_to_bev(const void* feat_split, const int32_t* coors, const int32_t* d_rows, int rows_cap, int C,
                            int D, int H, int W, int batch, void* bev_split, int32_t* tile_dist, sassd_stream_t stream);
                            /* tile_dist: optional, pre-filled with a large value (sassd_conv2d_f16x3_occ) */

/* SparseConvTensor.dense() + view (cmn.py:112-114) into the NHWC BEV map the
 * neck consumes: bev[b, y, x, d*C + c] = feat[row, c]  (reference channel c*D+d;
 * the permutation is folded into the first BEV conv's weights).  The map must be
 * zeroed by the caller (cudaMemsetAsync). */
int sassd_sparse_to_bev(const float* feat, const int32_t* coors, const int32_t* d_rows, int rows_cap, int C,
                        int D, int H, int W, float* bev, sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * second_box_decode + get_guided_anchors (ssd_rotate_head.py:53-91,307-372):
 * head [batch,H,W,head_stride] NHWC holds conv_box | conv_cls | conv_dir_cls
 * channels back to back; anchors [n_anchors,7] in (class,y,x,rot) order, one table shared by the
 * batch (anchors_per_frame = 0) or one per frame [batch,n_anchors,7] (anchors_per_frame = 1, the
 * reference's signature: ssd_rotate_head.py:316 indexes anchors[i]);
 * mask [batch,n_anchors] uint8.  Per frame, in anchor order: keep mask &&
 * max_c sigmoid(cls) > thr, decode, flip direction.  Outputs (capacity k_cap per frame):
 * boxes [batch,k_cap,7], labels [batch,k_cap] i32, index [batch,k_cap] i32
 * (anchor id), d_k [batch].
 * ---------------------------------------------------------------------- */
size_t sassd_decode_select_workspace_bytes(int batch, int n_anchors);
int sassd_decode_select(const float* head, int head_stride, int batch, int H, int W, int num_class,
                        const float* anchors, int anchors_per_frame, const uint8_t* mask, int n_anchors, float thr,
                        float* boxes, int32_t* labels, int32_t* index, int32_t* d_k, int k_cap,
                        int32_t* d_status, void* ws, size_t ws_bytes, sassd_stream_t stream);

/* PSWarpHead sampling (ssd_rotate_head.py:374-414,431-447): feat [batch,H,W,feat_stride]
 * NHWC with >= num_parts channels; part p = i*7+j samples channel p bilinearly at
 * the (i,j) tap of the 4x7 window of each guided box; score = mean over parts (logit). */
int sassd_pswarp(const float* feat, int feat_stride, int batch, int H, int W, const float* boxes,
                 const int32_t* d_k, int k_cap, float off_x, float off_y, float spatial_scale,
                 float* scores, sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * get_rescore_bboxes (ssd_rotate_head.py:487-533) = sigmoid(score) > score_thr,
 * boxes3d_to_bev_torch (iou3d_utils.py:47-60), nms_gpu (iou3d_utils.py:114-128,
 * iou3d.cpp:73-120, iou3d_kernel.cu:250-292) with the greedy sweep on the
 * device, gather.  Sort is stable (score descending, then candidate order).
 * det [batch,det_cap,9] = (x,y,z,w,l,h,ry,score,label); d_ndet [batch].
 * ---------------------------------------------------------------------- */
size_t sassd_rescore_nms_workspace_bytes(int batch, int k_cap, int nms_cap);
int sassd_rescore_nms(const float* boxes, const float* scores, const int32_t* labels, const int32_t* d_k,
                      int batch, int k_cap, float score_thr, float iou_thr, int nms_cap,
                      float* det, int32_t* d_ndet, int det_cap, int32_t* d_status,
                      void* ws, size_t ws_bytes, sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * KITTI result formatting of the NMS output, results.kitti_bbox2results
 * (transforms.py:225-279) for a whole batch.  det [batch,det_cap,9] and
 * d_ndet [batch] as written by sassd_rescore_nms; meta [batch][36] fp64 =
 * P2 (12), Tr_velo_to_cam (12), R0_rect (9), img_h, img_w, pad
 * (results.meta_block).  rows [batch,det_cap,14] fp64 = (alpha, bbox x1 y1 x2
 * y2, dimensions l h w, location x y z, rotation_y, score, label) of the boxes
 * whose image projection is not wholly outside the image, clipped to it, in
 * detection order; n_out [batch] their number.  Rows past n_out[b] are left
 * unwritten.  Arithmetic follows the host formatter's dtypes (fp32 yaw wrap,
 * corners and alpha; fp64 transforms and projection); sinf / cosf / atan2f and
 * the summation order of the host's matrix products differ, so the agreement
 * is within stated bounds, not bitwise.  No host synchronisation.
 * ---------------------------------------------------------------------- */
#define SASSD_KITTI_META 36
#define SASSD_KITTI_ROW 14
int sassd_kitti_format(const float* det, const int32_t* d_ndet, int batch, int det_cap, const double* meta,
                       double* rows, int32_t* n_out, sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * Detections of a set of single-class models (detectors.DetectorSet), one
 * block per frame.  Member m (m < n_members <= SASSD_MERGE_MAX) gives
 * host_dets[m] = det [batch,host_caps[m],9] and host_ndets[m] = d_ndet [batch]
 * as sassd_rescore_nms writes them (device pointers in host arrays).
 * det [batch,sum host_caps,9]: frame f holds member 0's first
 * min(d_ndet_0[f], cap_0) rows, then member 1's, ..., each copied bit for bit
 * but for its label (column 8), which gains host_label_offsets[m] (the
 * member's first class in the set's class list).  d_ndet [batch] = the
 * frame's row count.  Rows past it are left unwritten.  No NMS across
 * members, no host synchronisation: graph-capturable; sassd_kitti_format
 * then takes det_cap = sum host_caps.
 * ---------------------------------------------------------------------- */
#define SASSD_MERGE_MAX 16
int sassd_merge_detections(const float* const* host_dets, const int32_t* const* host_ndets, const int* host_caps,
                           const int* host_label_offsets, int n_members, int batch, float* det, int32_t* d_ndet,
                           sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * Auxiliary point-wise head, SpMiddleFHD.forward(is_test=False)
 * (cmn.py:121-135, :175-189): per voxel a foreground logit and a centre offset.
 *
 * sassd_three_nn: for every level-0 row r < *d_rows0 (mean [rows_cap0,4] =
 * SimpleVoxel mean x,y,z,r; coors0 [rows_cap0,4] (b,z,y,x)) the three nearest
 * centres of its own frame at each of the levels 1..3 (coorsL [capL,4], rows
 * sorted by flattened (b,z,y,x), *d_rowsL of them).  Centres are tensor2points
 * (transforms.py:218-223) with the reference's literal offset (0,-40,-3) and
 * voxel sizes (.1,.1,.2), (.2,.2,.4), (.4,.4,.8).  idx / dist2 [rows_cap0,3,3]
 * = (row, level, k): global row indices of the level and squared distances,
 * bit-identical to pointnet2 three_nn (interpolate_gpu.cu:9-56); a frame with
 * fewer than three centres gets idx 0 and dist2 +inf in the missing slots.
 * points_mean [rows_cap0,4] (may be NULL) receives (b, x, y, z), cmn.py:104-106.
 * Rows past *d_rows0 are left unwritten.
 *
 * sassd_point_aux_head: weights 1/(sqrt(dist2)+1e-8) normalised per level,
 * three_interpolate of each level's features, point_fc (160->64, no bias, no
 * activation), point_cls (64->1), point_reg (64->3), all fp32.  host_levels[3]
 * describe the features of levels 1..3 (32, 64, 64 channels): fp32 rows, or
 * split fp16 rows (hi plane, lo plane plane_stride elements further,
 * x = hi + lo * 2^-11).  w_fc_t = point_fc.weight^T [160,64]; w_out [4,64] =
 * point_cls.weight then point_reg.weight.  cls [rows_cap0], reg [rows_cap0,3].
 * Neither function synchronises with the host.
 * ---------------------------------------------------------------------- */
typedef struct {
    const void* rows;
    int64_t plane_stride;   /* split rows: elements from the hi to the lo plane */
    int32_t row_stride;     /* elements */
    int32_t channels;
    int32_t split;          /* 0: fp32 rows, 1: split fp16 rows */
    int32_t pad;
} sassd_point_levels;

int sassd_three_nn(const float* mean, const int32_t* coors0, const int32_t* d_rows0, int rows_cap0,
                   const int32_t* coors1, const int32_t* d_rows1, const int32_t* coors2, const int32_t* d_rows2,
                   const int32_t* coors3, const int32_t* d_rows3, int32_t* idx, float* dist2, float* points_mean,
                   sassd_stream_t stream);
int sassd_point_aux_head(const int32_t* idx, const float* dist2, const int32_t* d_rows0, int rows_cap0,
                         const sassd_point_levels* host_levels, const float* w_fc_t, const float* w_out, float* cls,
                         float* reg, sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * Training targets and losses, forward only, for labelled frames
 * (cmn.py:44-100, target_ops.py:139-277, ssd_rotate_head.py:237-305,450-485,
 * losses.py:31-114).  Ground truth per frame: gt [batch,gt_cap,7] boxes
 * (x, y, z_bottom, w, l, h, ry), d_ngt [batch] their number (more than
 * gt_cap sets SASSD_FLAG_GT_CAP; the first gt_cap are used), gt_cap <=
 * SASSD_GT_CAP_MAX.  A frame without GT is all background.  No host
 * synchronisation; workspace: sassd_loss_workspace_bytes(batch, gt_cap).
 * Loss sums are fp32 per element, fp64 across elements, reduced in a fixed
 * order: the same inputs give the same bits.
 *
 * sassd_points_in_boxes: pts_in_boxes3d of each voxel row r < *d_rows
 * (points_mean [rows_cap,4] = (b, x, y, z)) against its frame's boxes with
 * the reference's C++ expression types.  labels [rows_cap] = 1 inside any
 * box, offsets [rows_cap,3] = point - centre of the LAST containing box in
 * box order (z centre = z_bottom + fourth value / 2, as points_op.cpp:139),
 * 0 when none; *d_npos = number of labelled rows.
 *
 * sassd_assign_rpn: create_target_torch with NearestIouSimilarity per frame
 * and class.  anchors [n_anchors,7] (shared) or [batch,n_anchors,7], classes
 * concatenated (n_anchors / num_class each), mask [batch,n_anchors];
 * gt_class [batch,gt_cap] = anchor class of each GT (-1: none), gt_label =
 * the label a positive gets; host_pos_thr / host_neg_thr [num_class],
 * num_class <= 8.  labels [batch,n_anchors] (-1 unmasked / ignored, 0
 * background, > 0 positive), targets [batch,n_anchors,7] second_box_encode
 * for the positives (0 elsewhere), ious (may be NULL) = anchor_to_gt_max
 * (0 unmasked), d_npos [batch] positives per frame.
 *
 * sassd_assign_pswarp: the same rules with RotateIou3dSimilarity, every
 * label 1 and no mask, over box slots [batch,n_box,7]: slots [0, head_cap)
 * hold d_head[b] boxes (the GT rows of the guided list; d_head may be NULL
 * when head_cap is 0) and slots [head_cap, n_box) hold d_k[b] boxes.
 * labels [batch,n_box] (-1 in empty slots), ious, d_npos [batch].
 *
 * sassd_rpn_loss: out[3] = rpn_loc_loss, rpn_cls_loss, rpn_dir_loss
 * (NormByNumPositives per frame, / batch, x2 and x0.2) from the head map of
 * sassd_decode_select and the labels / targets / d_npos of sassd_assign_rpn.
 * sassd_pswarp_loss: out[1] = loss_cls, focal loss over scores
 * [batch,n_box] normalised by the positives of the whole batch, / batch.
 * sassd_aux_loss: out[2] = aux_loss_cls, aux_loss_reg from point_cls
 * [rows_cap], point_reg [rows_cap,3] and sassd_points_in_boxes' outputs.
 * ---------------------------------------------------------------------- */
#define SASSD_GT_CAP_MAX 256
size_t sassd_loss_workspace_bytes(int batch, int gt_cap);
int sassd_points_in_boxes(const float* points_mean, const int32_t* d_rows, int rows_cap, const float* gt,
                          const int32_t* d_ngt, int batch, int gt_cap, int32_t* labels, float* offsets,
                          int32_t* d_npos, int32_t* d_status, sassd_stream_t stream);
int sassd_assign_rpn(const float* anchors, int anchors_per_frame, const uint8_t* mask, int n_anchors, int num_class,
                     const float* gt, const int32_t* gt_class, const int32_t* gt_label, const int32_t* d_ngt,
                     int batch, int gt_cap, const float* host_pos_thr, const float* host_neg_thr, int32_t* labels,
                     float* targets, float* ious, int32_t* d_npos, int32_t* d_status, void* ws, size_t ws_bytes,
                     sassd_stream_t stream);
int sassd_assign_pswarp(const float* gt, const int32_t* d_ngt, int batch, int gt_cap, const float* boxes, int n_box,
                        const int32_t* d_head, int head_cap, const int32_t* d_k, float pos_thr, float neg_thr,
                        int32_t* labels, float* ious, int32_t* d_npos, int32_t* d_status, void* ws,
                        size_t ws_bytes, sassd_stream_t stream);
int sassd_rpn_loss(const float* head, int head_stride, int batch, int H, int W, int num_class, const float* anchors,
                   int anchors_per_frame, int n_anchors, const int32_t* labels, const float* targets,
                   const int32_t* d_npos, float* out, void* ws, size_t ws_bytes, sassd_stream_t stream);
int sassd_pswarp_loss(const float* scores, const int32_t* labels, int batch, int n_box, const int32_t* d_npos,
                      float* out, void* ws, size_t ws_bytes, sassd_stream_t stream);
int sassd_aux_loss(const float* point_cls, const float* point_reg, const int32_t* labels, const float* offsets,
                   const int32_t* d_rows, int rows_cap, int batch, const int32_t* d_npos, float* out, void* ws,
                   size_t ws_bytes, sassd_stream_t stream);

/* iou3d_cuda.nms_gpu alone (iou3d.cpp:73-120): boxes [n,5] already sorted by
 * score; mask [n, ceil(n/64)] u64 in the reference layout (only columns j > i
 * are filled; the reference also fills the unused lower triangle); keep [n]
 * int64 indices, *d_nkeep their number. */
size_t sassd_nms_workspace_bytes(int n);
int sassd_nms_mask(const float* boxes5, int n, float thr, uint64_t* mask, sassd_stream_t stream);
int sassd_nms_sorted(const float* boxes5, int n, float thr, int64_t* keep, int32_t* d_nkeep,
                     void* ws, size_t ws_bytes, sassd_stream_t stream);
/* iou3d_cuda.boxes_iou_bev_gpu (iou3d.cpp:52-71): dense [na, nb] rotated BEV IoU. */
int sassd_boxes_iou_bev(const float* boxes_a, int na, const float* boxes_b, int nb, float* iou, sassd_stream_t stream);

/* ---- KITTI evaluation support (SURVEY.md section 8 row f4) ----------------------------------------------------
 * Rotated-box overlap of the reference's evaluator (mmdet/core/post_processing/rotate_nms_gpu.py:536-627
 * rotate_iou_gpu_eval), batched over frames: boxes / query are concatenated [sum, 5] (x, y, dx, dy, angle) arrays
 * with per-frame offsets [nframes + 1]; out[out_off[f] + n * nq_f + k] = overlap(box n, query k) of frame f.
 * criterion: -1 IoU, 0 intersection / area(query), 1 intersection / area(box), 2 intersection area. */
int sassd_rotate_overlap_eval(const float* boxes, const int32_t* box_off, const float* query, const int32_t* query_off,
                              const int64_t* out_off, int nframes, int criterion, int max_pairs_per_frame, float* out,
                              sassd_stream_t stream);
/* HOST function (all pointers are host memory): greedy GT<->detection matching of the KITTI protocol
 * (mmdet/core/evaluation/kitti_eval.py:164-283, :295-342).  nthresh == 0: collect the scores of the true positives
 * (tp_scores capacity = number of gt rows); nthresh > 0: pr[t] += (tp, fp, fn, similarity) for every threshold. */
int sassd_kitti_match(int nframes, const double* overlaps, const int64_t* ov_off, const int32_t* gt_off,
                      const int32_t* dt_off, const int32_t* dc_off, const double* gt_alpha, const double* dt_alpha,
                      const double* dt_score, const double* dt_bbox, const double* dc_bbox, const int32_t* ign_gt,
                      const int32_t* ign_dt, int metric, double min_overlap, int compute_aos, int nthresh,
                      const double* thresholds, double* pr, double* tp_scores, int64_t* n_tp_scores);
/* HOST function: the same matching's assignment for sassd_kitti_eval_assign's table, one (class, difficulty, metric)
 * of one set (compute_fp=True at a threshold below every score): gt_det[row] the matched detection's row or -1,
 * gt_ov[row] their overlap (0 when unmatched), dt_state[row] SASSD_KITTI_DT_* of every detection row. */
int sassd_kitti_assign(int nframes, const double* overlaps, const int64_t* ov_off, const int32_t* gt_off,
                       const int32_t* dt_off, const int32_t* dc_off, const double* dt_score, const double* dt_bbox,
                       const double* dc_bbox, const int32_t* ign_gt, const int32_t* ign_dt, int metric,
                       double min_overlap, int32_t* gt_det, double* gt_ov, int8_t* dt_state);

/* The same cleaning and matching on the device (csrc/kitti_match.cu), for K detection sets against one GT and any
 * number of min-overlap rows, with no per-frame host work.  GT rows of all frames are concatenated (gt_off
 * [nframes + 1]); detection rows of set k's frame f are [dt_off[k * nframes + f], dt_off[k * nframes + f + 1]).
 * Name ids: each distinct lower-cased class name has one id (-1 for names of no class).
 *
 * sassd_kitti_eval_flags: clean_data's flags for every (class c, difficulty entry d), cd = c * ndiff + d:
 * ign_gt[cd * ngt + row] (0 evaluate, 1 ignore, -1 other class), ign_dt[cd * ndt + row] (1 too low, 0 the class,
 * -1 other) and n_valid[cd] += the rows flagged 0 (zero it first).  classes[2c] = class c's name id, classes[2c+1] the
 * id of the name counted as ignored for it (van for car, person_sitting for pedestrian) or -1; limits[3d .. 3d+2] =
 * (max occlusion, max truncation, min height) of difficulty entry d.  All pointers are device memory. */
int sassd_kitti_eval_flags(int ngt, const int32_t* gt_name, const double* gt_occ, const double* gt_trunc,
                           const double* gt_bbox, int ndt, const int32_t* dt_name, const double* dt_bbox, int nclass,
                           const int32_t* classes, int ndiff, const double* limits, int8_t* ign_gt, int8_t* ign_dt,
                           int32_t* n_valid, sassd_stream_t stream);
/* sassd_kitti_eval_flags with a range bin per difficulty entry.  A row's range is its ground distance from the camera,
 * sqrt(x * x + z * z) of its camera-frame location (gt_cam / dt_cam rows x, y, z, l, h, w, ry; fp64).  Entry d keeps
 * the rows with ranges[2d] <= range < ranges[2d+1]: a GT row of the class outside it is flagged 1 (ignored, as a GT
 * harder than the difficulty is), a detection of the class outside it 1 (as a low one is); other classes and DontCare
 * rows are not range-tested, and a NaN range falls in no bin.  ranges null, or an entry whose lower edge is -inf, means
 * no range test.  gt_range / dt_range, when not null, receive every row's range.  With ranges null and no range
 * outputs this is sassd_kitti_eval_flags, which calls it so. */
int sassd_kitti_eval_flags_ranged(int ngt, const int32_t* gt_name, const double* gt_occ, const double* gt_trunc,
                                  const double* gt_bbox, const double* gt_cam, int ndt, const int32_t* dt_name,
                                  const double* dt_bbox, const double* dt_cam, int nclass, const int32_t* classes,
                                  int ndiff, const double* limits, const double* ranges, int8_t* ign_gt,
                                  int8_t* ign_dt, int32_t* n_valid, double* gt_range, double* dt_range,
                                  sassd_stream_t stream);
/* The bbox, BEV and 3-D overlap matrices of every (set, frame) block b = k * nframes + f, row-major [detection, GT]
 * at ov_off[b] (fp64, bit for bit the host's image_box_overlap / float32 BEV IoU / _d3_from_bev).  bev_iou and
 * bev_inter are sassd_rotate_overlap_eval's criterion -1 and 2 outputs over the same blocks; cam rows are
 * (x, y, z, l, h, w, ry) in the camera frame. */
int sassd_kitti_eval_overlaps(int nsets, int nframes, const int32_t* gt_off, const int32_t* dt_off,
                              const int64_t* ov_off, const double* gt_cam, const double* dt_cam, const double* gt_bbox,
                              const double* dt_bbox, const float* bev_iou, const float* bev_inter,
                              int max_pairs_per_frame, double* ov_bbox, double* ov_bev, double* ov_3d,
                              sassd_stream_t stream);
/* HOST function: aos[ov_off[b] + j * ng + i] = (1 + cos(gt_alpha[i] - dt_alpha[j])) / 2 with the host matcher's cos. */
int sassd_kitti_aos_table(int nsets, int nframes, const int32_t* gt_off, const int32_t* dt_off, const int64_t* ov_off,
                          const double* gt_alpha, const double* dt_alpha, double* aos);

typedef struct {
    int nsets, nframes, nclass, ndiff, nover;     /* K, frames, classes, difficulty entries, min-overlap rows */
    int max_nd, max_ng;                           /* most detections / GT rows of one frame */
    const int32_t *gt_off, *dt_off;
    const int64_t* ov_off;
    const int32_t* gt_dc;                         /* 1 for DontCare GT rows */
    const double *gt_bbox, *dt_bbox, *dt_score;
    const double *ov_bbox, *ov_bev, *ov_3d;       /* sassd_kitti_eval_overlaps */
    const double* aos_table;                      /* sassd_kitti_aos_table, or null */
    const int32_t* compute_aos;                   /* [nsets] */
    const double* min_overlaps;                   /* [nover, 3 metrics, nclass] */
    const int8_t *ign_gt, *ign_dt;
    const int32_t* n_valid;                       /* sassd_kitti_eval_flags */
    const int64_t* score_off;                     /* [jobs + 1]: power-of-two region per job, >= n_valid of its cd */
} SassdKittiEvalDesc;
/* Job = (((k * nclass + c) * ndiff + d) * 3 + metric) * nover + o.  For every job: the true-positive scores
 * (compute_fp=False) into scores[score_off[job] ..], n_scores[job] of them; the thresholds of get_thresholds,
 * thresholds[job * 41 + t] for t < n_thresh[job]; and pr[(job * 41 + t) * 4 + (tp, fp, fn, similarity)] summed over
 * the frames as fused_compute_statistics does (the similarity in frame order).  Rows past n_thresh are zero.
 * ws: sassd_kitti_eval_workspace_bytes(max_nd, max_ng) bytes.  SASSD_ERR_ARG for negative counts or a job grid past
 * 2^31 (job, threshold) items. */
size_t sassd_kitti_eval_workspace_bytes(int max_nd, int max_ng);
int sassd_kitti_eval_match(const SassdKittiEvalDesc* desc, double* scores, int32_t* n_scores, double* thresholds,
                           int32_t* n_thresh, double* pr, void* ws, size_t ws_bytes, sassd_stream_t stream);

/* Match-table states of a detection row (compute_statistics_jit's fate of the detection). */
#define SASSD_KITTI_DT_NOT_COUNTED 0   /* flag -1 (other class) or 1 (ignored) and not assigned */
#define SASSD_KITTI_DT_TP 1            /* true positive */
#define SASSD_KITTI_DT_FP 2            /* false positive */
#define SASSD_KITTI_DT_DONTCARE 3      /* unassigned, inside a DontCare area (bbox metric only): not a false positive */
#define SASSD_KITTI_DT_IGNORED 4       /* assigned to an ignored GT, or an ignored detection assigned to a GT */

/* The match table: compute_statistics_jit's assignment (compute_fp=True at a threshold below every score, so every
 * detection counts) for every (set k, class c, difficulty entry d < ndiff, metric m) at min-overlap row `row` of the
 * desc (whose flags and overlaps it reads; aos_table, compute_aos, n_valid and score_off are not read).  With G / D the
 * GT / detection rows of all sets:
 *   gt_det[(((k * nclass + c) * ndiff + d) * 3 + m) * G + i]   the matched detection's row within set k, or -1;
 *   gt_ov[same]                                                  their overlap, 0 when unmatched;
 *   dt_state[((c * ndiff + d) * 3 + m) * D + j]                  SASSD_KITTI_DT_* of detection row j;
 *   tp_err[(((k * nclass + c) * ndiff + d) * G + i) * 3 + e]     the 3-D metric's TP errors (ATE, ASE, AOE) of GT row
 *                                                                i, NaN when it has no true positive there.
 * ATE = sqrt(dx * dx + dz * dz) of the camera-frame centres (detection minus GT); ASE = 1 - vi / ((vg + vd) - vi) with
 * vi = (min l * min h) * min w and vg, vd = (l * h) * w; AOE = min(|w|, pi) with dr = ry_det - ry_gt and
 * w = dr - 2pi * floor((dr + pi) / 2pi).  All fp64, rounded operation by operation.  gt_cam / dt_cam are the camera
 * rows of the flags.  ws as sassd_kitti_eval_match's. */
int sassd_kitti_eval_assign(const SassdKittiEvalDesc* desc, int row, int ndiff, const double* gt_cam,
                            const double* dt_cam, int32_t* gt_det, double* gt_ov, int8_t* dt_state, double* tp_err,
                            void* ws, size_t ws_bytes, sassd_stream_t stream);

/* KITTI label / result files parsed on the device (csrc/kitti_parse.cu), get_label_anno's semantics
 * (tools/kitti_common.py:560-601).  buf holds every file's bytes back to back, file f at [file_off[f], file_off[f+1])
 * (int64).  All pointers are device memory.
 *
 * sassd_kitti_scan_labels: per file, n_lines[f] its readlines() line count ('\n' ends a line) and flags[f]:
 * SASSD_KITTI_PARSE_SCORE when its first line has exactly 16 space-separated fields, SASSD_KITTI_PARSE_DEFER when the
 * file is outside the device grammar (a byte >= 0x80 or a control character, an empty field, a missing converted field,
 * a number outside [+-]?digits[.digits][(e|E)[+-]?digits], with more than 19 significant digits, a significand >= 2^53
 * or a decimal exponent beyond +-22, an occluded value beyond int64) and must be read on the host (n_lines[f] = 0).
 *
 * sassd_kitti_parse_labels: the rows of every file not deferred, file f's lines at rows row_off[f] .. (row_off [nfiles
 * + 1], nrows = row_off[nfiles]; a deferred file's rows are left unwritten): name_id (the index of the lower-cased name
 * in the table names / name_off [nnames + 1], or -1), dontcare (name == "DontCare"), truncated, occluded
 * (int(float(x)) as fp64), alpha, bbox [rows, 4], cam [rows, 7] (location, the file's h, w, l as l, h, w, rotation_y)
 * and score (the 16th field with SASSD_KITTI_PARSE_SCORE, else 0), each equal to Python's float() bit for bit.
 * ws: sassd_kitti_parse_workspace_bytes(nrows) bytes. */
#define SASSD_KITTI_PARSE_DEFER 1
#define SASSD_KITTI_PARSE_SCORE 2
int sassd_kitti_scan_labels(const uint8_t* buf, const int64_t* file_off, int nfiles, int32_t* n_lines, int32_t* flags,
                            sassd_stream_t stream);
size_t sassd_kitti_parse_workspace_bytes(int nrows);
int sassd_kitti_parse_labels(const uint8_t* buf, const int64_t* file_off, int nfiles, const int32_t* flags,
                             const int32_t* row_off, int nrows, const char* names, const int32_t* name_off, int nnames,
                             int32_t* name_id, int32_t* dontcare, double* truncated, double* occluded, double* alpha,
                             double* bbox, double* cam, double* score, void* ws, size_t ws_bytes,
                             sassd_stream_t stream);

/* ------------------------------------------------------------------------
 * Training-time augmentation (the reference's PointAugmentor as
 * prepare_train_img applies it, mmdet/core/point_cloud/point_augmentor.py,
 * mmdet/datasets/kitti.py:181-209).  The host draws every random number and
 * computes the box geometry; boxes of frame b are [d_box_off[b], d_box_off[b+1]).
 *
 * sassd_augment_drop_points: sassd_frustum_crop's compaction, keeping the
 * points of frame b outside every box of frame b, under the reference's plane
 * test in fp32 (planes [boxes][6][4] fp32, `s >= 0` rejects).  Workspace:
 * sassd_frustum_crop_workspace_bytes.
 *
 * sassd_augment_noise_search: noise_per_box, one CTA per frame.  boxes
 * [boxes][5] fp32 (x, y, w, l, ry), box_trig [boxes][2] (cosf, sinf of ry),
 * try_trig [boxes][tries][2] (cos, sin of each try's rotation, rounded to
 * fp32), loc [boxes][tries][3] fp64 location noise.  sel[k] = the smallest
 * try whose BEV box collides with no other box's current corners (a box fully
 * inside another collides), or -1.  Boxes of a frame past SASSD_GT_CAP_MAX
 * get -1 and set SASSD_FLAG_GT_CAP.  tries <= 128.
 *
 * sassd_augment_assemble: per frame, the database rows of its sampled
 * records (records s in [d_srow_off..] order: rows db[d_srec_db[s] ..] of
 * count d_srec_off[s+1] - d_srec_off[s], each x, y, z plus srec_ctr[s] fp64,
 * then, when srec_dz [n_rec] is not null, z minus srec_dz[s] fp64, rounded
 * again: the record's move onto the frame's road plane; null: no move, and
 * a non-null srec_dz needs n_rec > 0) followed by the rows sassd_augment_drop_points kept; each row then takes
 * the transform of the first box whose fp32 planes contain it (centres
 * [boxes][3] fp32, its try sel[k]), the frame's flip, rotation and scale
 * (frame_tf [batch][6]: flip, R00, R01, R10, R11, scale).  More than out_cap
 * rows: the rest are not written and SASSD_FLAG_POINTS_CAP is set
 * (d_pt_off_out stays exact).  batch <= 256.
 * ---------------------------------------------------------------------- */
int sassd_augment_drop_points(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch,
                              const float* planes, const int32_t* d_box_off, float* points_out,
                              int32_t* d_pt_off_out, void* ws, size_t ws_bytes, sassd_stream_t stream);
int sassd_augment_noise_search(const float* boxes, const float* box_trig, const int32_t* d_box_off, int batch,
                               int tries, const float* try_trig, const double* loc, int32_t* sel,
                               int32_t* d_status, sassd_stream_t stream);
int sassd_augment_assemble(const float* kept, const int32_t* d_kept_off, int batch, const int32_t* d_srow_off,
                           const int32_t* d_srec_off, int n_rec, const int32_t* d_srec_db, const double* srec_ctr,
                           const double* srec_dz, const float* db, const int32_t* d_box_off, const float* planes, const float* centres,
                           const int32_t* sel, int tries, const float* try_trig, const double* loc,
                           const float* frame_tf, int out_cap, float* points_out, int32_t* d_pt_off_out,
                           int32_t* d_status, sassd_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SASSD_B200_H */

// Training targets and losses of SA-SSD, forward only (no autograd), for labelled frames.
//
// Replaces, on the device and for the whole batch at once:
//  * SpMiddleFHD.build_aux_target / pts_in_boxes3d (cmn.py:44-70, points_op.cpp:92-144), a host double loop per frame;
//  * create_target_torch (target_ops.py:139-277) with NearestIouSimilarity (SSDRotateHead.loss, per frame and class)
//    and RotateIou3dSimilarity (PSWarpHead.loss), which builds the dense anchors x GT IoU matrix and syncs on
//    nonzero();
//  * the losses of SSDRotateHead.loss, PSWarpHead.loss and SpMiddleFHD.aux_loss (ssd_rotate_head.py:237-305,450-485,
//    cmn.py:72-100, losses.py:31-114).
//
// The assignment never materialises the IoU matrix: one kernel runs twice over the anchors.  Phase 0 reduces the
// per-GT maximum (shared-memory, then global atomicMax on the bits of the non-negative float); phase 1 recomputes every
// IoU with the same instructions, so ties compare bit-identical values, and writes labels and box targets.  Losses are
// fp32 per element, summed in fp64 per block and then by one final block in a fixed order (no float atomics), so the
// same inputs give the same bits on every call.  Integer atomics count positives.
#include "common.cuh"
#include "box_overlap.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxClasses = 8;
constexpr int kSlots = 4;               // loss partial sums per block
constexpr float kPiF = 3.14159274101257324f;          // (float)M_PI
constexpr float kQuarterPiF = 0.785398185253143311f;  // (float)(M_PI / 4)

// ---------------------------------------------------------------------------------------------------- aux targets
// pt_in_box3d_cpu (points_op.cpp:92-105) with its expression types: h/2.0, w/2.0, l/2.0 are double, cz is rounded to
// float, cos / sin are double stored to float, and the rotation is fp32 without contraction (the reference is x86
// C++ built without FMA).
__device__ __forceinline__ bool pt_in_box(float x, float y, float z, const float* b) {
    const float cx = b[0], cy = b[1], bottom_z = b[2], w = b[3], l = b[4], h = b[5], angle = b[6];
    const float max_dis = 10.0f;
    const float cz = (float)((double)bottom_z + (double)h / 2.0);
    if ((fabsf(__fsub_rn(x, cx)) > max_dis) || ((double)fabsf(__fsub_rn(z, cz)) > (double)h / 2.0) ||
        (fabsf(__fsub_rn(y, cy)) > max_dis))
        return false;
    const float cosa = (float)cos((double)angle), sina = (float)sin((double)angle);
    const float dx = __fsub_rn(x, cx), dy = __fsub_rn(y, cy);
    const float x_rot = __fadd_rn(__fmul_rn(dx, cosa), __fmul_rn(dy, -sina));
    const float y_rot = __fadd_rn(__fmul_rn(dx, sina), __fmul_rn(dy, cosa));
    return ((double)x_rot >= -(double)w / 2.0) & ((double)x_rot <= (double)w / 2.0) &
           ((double)y_rot >= -(double)l / 2.0) & ((double)y_rot <= (double)l / 2.0);
}

__global__ void __launch_bounds__(kThreads)
points_in_boxes_kernel(const float* __restrict__ pm, const int* __restrict__ d_rows, int rows_cap,
                       const float* __restrict__ gt, const int* __restrict__ d_ngt, int batch, int gt_cap,
                       int* __restrict__ labels, float* __restrict__ offsets, int* __restrict__ d_npos) {
    const int rows = min(d_rows[0], rows_cap);
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r - (int)threadIdx.x < rows; r += gridDim.x * blockDim.x) {
        int lab = 0;
        if (r < rows) {
            const int b = (int)pm[(size_t)r * 4];
            const float x = pm[(size_t)r * 4 + 1], y = pm[(size_t)r * 4 + 2], z = pm[(size_t)r * 4 + 3];
            float o0 = 0.f, o1 = 0.f, o2 = 0.f;
            if (b >= 0 && b < batch) {
                const int n = min(d_ngt[b], gt_cap);
                const float* g = gt + (size_t)b * gt_cap * 7;
                for (int j = 0; j < n; ++j) {
                    const float* bj = g + j * 7;
                    if (pt_in_box(x, y, z, bj)) {      // the label is the max over boxes, the offset the last box's
                        lab = 1;
                        o0 = __fsub_rn(x, bj[0]);
                        o1 = __fsub_rn(y, bj[1]);
                        // points_op.cpp:139 reads the box's fourth value (w in this format) as the height
                        o2 = (float)((double)z - ((double)bj[2] + (double)bj[3] / 2.0));
                    }
                }
            }
            labels[r] = lab;
            offsets[(size_t)r * 3] = o0;
            offsets[(size_t)r * 3 + 1] = o1;
            offsets[(size_t)r * 3 + 2] = o2;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, lab);
        if ((threadIdx.x & 31) == 0 && bal) atomicAdd(d_npos, __popc(bal));
    }
}

// ---------------------------------------------------------------------------------------------------- assignment
struct AssignParams {
    int mode;                       // 0: RPN, NearestIouSimilarity per class; 1: PSWarp, RotateIou3dSimilarity
    int batch, gt_cap, n;           // n: anchors (RPN) or box slots (PSWarp) per frame
    const float* gt;                // [batch, gt_cap, 7]
    const int* gt_class;            // [batch, gt_cap] anchor class of each GT (-1: none); RPN only
    const int* gt_label;            // [batch, gt_cap] label written for a positive; RPN only (PSWarp: 1)
    const int* d_ngt;               // [batch]
    // RPN
    const float* anchors;           // [n, 7] or [batch, n, 7]
    int anchors_per_frame, num_class, per_class;
    const uint8_t* mask;            // [batch, n]
    float pos_thr[kMaxClasses], neg_thr[kMaxClasses];
    // PSWarp: box slots [0, head_cap) hold d_head[b] boxes, slots [head_cap, n) hold d_k[b] boxes
    const float* boxes;             // [batch, n, 7]
    const int* d_head;              // may be NULL (no head segment)
    const int* d_k;
    int head_cap;
    // outputs
    int* labels;                    // [batch, n]
    float* targets;                 // [batch, n, 7] (RPN; may be NULL)
    float* ious;                    // [batch, n] anchor_to_gt_max (0 where not assigned; may be NULL)
    int* npos;                      // [batch]
    int* gmax;                      // [batch, gt_cap] workspace: float bits of the per-GT maximum
};

// boxes3d_to_near_torch (iou3d_utils.py:8-26) in fp32: limit_period, the > pi/4 swap, centre -/+ half size.
__device__ __forceinline__ void near_box(const float* b, float* q) {
    const float rot = b[6];
    const float lp = __fsub_rn(rot, __fmul_rn(floorf(__fadd_rn(__fdiv_rn(rot, kPiF), 0.5f)), kPiF));
    const bool swap = fabsf(lp) > kQuarterPiF;
    const float dx = swap ? b[4] : b[3], dy = swap ? b[3] : b[4];
    q[0] = __fsub_rn(b[0], dx / 2.f);
    q[1] = __fsub_rn(b[1], dy / 2.f);
    q[2] = __fadd_rn(b[0], dx / 2.f);
    q[3] = __fadd_rn(b[1], dy / 2.f);
}

// boxes_iou(mode='iou', eps=0) of two near boxes (iou3d_utils.py:28-45), each operation rounded on its own.
__device__ __forceinline__ float near_iou(const float* a, const float* g) {
    const float w = fmaxf(__fsub_rn(fminf(a[2], g[2]), fmaxf(a[0], g[0])), 0.f);
    const float h = fmaxf(__fsub_rn(fminf(a[3], g[3]), fmaxf(a[1], g[1])), 0.f);
    const float ov = __fmul_rn(w, h);
    const float area1 = __fmul_rn(__fsub_rn(a[2], a[0]), __fsub_rn(a[3], a[1]));
    const float area2 = __fmul_rn(__fsub_rn(g[2], g[0]), __fsub_rn(g[3], g[1]));
    return __fdiv_rn(ov, __fsub_rn(__fadd_rn(area1, area2), ov));
}

// boxes3d_to_bev_torch (iou3d_utils.py:47-60): (x - b3/2, y - b4/2, x + b3/2, y + b4/2, ry).
__device__ __forceinline__ void bev_box(const float* b, float* q) {
    q[0] = __fsub_rn(b[0], b[3] / 2.f);
    q[1] = __fsub_rn(b[1], b[4] / 2.f);
    q[2] = __fadd_rn(b[0], b[3] / 2.f);
    q[3] = __fadd_rn(b[1], b[4] / 2.f);
    q[4] = b[6];
}

// boxes_iou3d_gpu (iou3d_utils.py:79-111): rotated BEV overlap (box_overlap) x bottom-based height overlap over
// clamp(vol_a + vol_b - overlap, 1e-7).  a = the box being assigned, g = the GT (the reference's argument order).
__device__ __forceinline__ float iou3d(const float* a, const float* qa, const float* g, const float* qg) {
    const float bev = rotated_overlap(qa, qg);
    const float top = fminf(__fadd_rn(a[2], a[5]), __fadd_rn(g[2], g[5]));
    const float oh = fmaxf(__fsub_rn(top, fmaxf(a[2], g[2])), 0.f);
    const float ov = __fmul_rn(bev, oh);
    const float va = __fmul_rn(__fmul_rn(a[3], a[4]), a[5]);
    const float vg = __fmul_rn(__fmul_rn(g[3], g[4]), g[5]);
    return __fdiv_rn(ov, fmaxf(__fsub_rn(__fadd_rn(va, vg), ov), 1e-7f));
}

// second_box_encode (ssd_rotate_head.py:15-51) in fp32: z to the centre, offsets over the anchor diagonal, log sizes.
__device__ __forceinline__ void box_encode(const float* g, const float* a, float* t) {
    const float zg = __fadd_rn(g[2], g[5] / 2.f), za = __fadd_rn(a[2], a[5] / 2.f);
    const float diag = sqrtf(__fadd_rn(__fmul_rn(a[4], a[4]), __fmul_rn(a[3], a[3])));
    t[0] = __fdiv_rn(__fsub_rn(g[0], a[0]), diag);
    t[1] = __fdiv_rn(__fsub_rn(g[1], a[1]), diag);
    t[2] = __fdiv_rn(__fsub_rn(zg, za), a[5]);
    t[3] = logf(__fdiv_rn(g[3], a[3]));
    t[4] = logf(__fdiv_rn(g[4], a[4]));
    t[5] = logf(__fdiv_rn(g[5], a[5]));
    t[6] = __fsub_rn(g[6], a[6]);
}

__global__ void __launch_bounds__(kThreads) assign_kernel(const AssignParams p, int phase) {
    extern __shared__ float smem[];
    const int b = blockIdx.y, G = p.gt_cap;
    float* s_gt = smem;                                   // [G][7]
    float* s_q = s_gt + G * 7;                            // [G][5] near or BEV box
    int* s_cls = (int*)(s_q + G * 5);
    int* s_lab = s_cls + G;
    int* s_max = s_lab + G;
    const int ngt = min(p.d_ngt[b], G);
    for (int j = threadIdx.x; j < ngt; j += blockDim.x) {
        const float* g = p.gt + ((size_t)b * G + j) * 7;
        for (int e = 0; e < 7; ++e) s_gt[j * 7 + e] = g[e];
        if (p.mode == 0) near_box(s_gt + j * 7, s_q + j * 5);
        else bev_box(s_gt + j * 7, s_q + j * 5);
        s_cls[j] = p.mode == 0 ? p.gt_class[(size_t)b * G + j] : 0;
        s_lab[j] = p.mode == 0 ? p.gt_label[(size_t)b * G + j] : 1;
        s_max[j] = phase == 0 ? 0 : p.gmax[(size_t)b * G + j];
    }
    __syncthreads();
    int nhead = 0, nk = 0;
    if (p.mode == 1) {
        nhead = p.d_head ? min(p.d_head[b], p.head_cap) : 0;
        nk = min(p.d_k[b], p.n - p.head_cap);
    }
    int my_pos = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
        const size_t o = (size_t)b * p.n + i;
        const float* a;
        int c = 0;
        bool valid;
        float qa[5];
        if (p.mode == 0) {
            c = i / p.per_class;
            valid = p.mask[o] != 0;
            a = p.anchors + ((p.anchors_per_frame ? o : (size_t)i) * 7);
        } else {
            valid = i < nhead || (i >= p.head_cap && i - p.head_cap < nk);
            a = p.boxes + o * 7;
        }
        if (!valid) {
            if (phase == 1) {
                p.labels[o] = -1;
                if (p.targets) for (int e = 0; e < 7; ++e) p.targets[o * 7 + e] = 0.f;
                if (p.ious) p.ious[o] = 0.f;
            }
            continue;
        }
        float ab[7];
        for (int e = 0; e < 7; ++e) ab[e] = a[e];
        if (p.mode == 0) near_box(ab, qa);
        else bev_box(ab, qa);
        float best = 0.f;
        int arg = -1;
        bool forced = false;
        for (int j = 0; j < ngt; ++j) {
            if (s_cls[j] != c) continue;
            const float v = p.mode == 0 ? near_iou(qa, s_q + j * 5) : iou3d(ab, qa, s_gt + j * 7, s_q + j * 5);
            if (arg < 0 || v > best) { best = v; arg = j; }     // argmax: the first maximum
            if (phase == 0) {
                if (v > 0.f) atomicMax(&s_max[j], __float_as_int(v));
            } else {
                // a GT whose maximum is 0 gets -1 (target_ops.py:211-212) and forces nothing
                const int m = s_max[j];
                forced |= m > 0 && v == __int_as_float(m);
            }
        }
        if (phase == 0) continue;
        int label;
        bool fg = false;
        if (arg < 0) {              // no GT of this class in the frame: every cared anchor is background
            label = 0;
            best = 0.f;
        } else {
            const int lab = s_lab[arg];
            const float pos = p.mode == 0 ? p.pos_thr[c] : p.pos_thr[0];
            const float neg = p.mode == 0 ? p.neg_thr[c] : p.neg_thr[0];
            // write order of target_ops.py:213-251: forced, >= pos, < neg -> 0, forced again
            label = -1;
            if (forced || best >= pos) label = lab;
            fg = label > 0;         // fg_inds are taken before the background write
            if (best < neg) label = 0;
            if (forced) label = lab;
        }
        p.labels[o] = label;
        if (p.ious) p.ious[o] = best;
        if (p.targets) {
            float t[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (fg) box_encode(s_gt + arg * 7, ab, t);
            for (int e = 0; e < 7; ++e) p.targets[o * 7 + e] = t[e];
        }
        my_pos += label > 0;
    }
    if (phase == 0) {
        __syncthreads();
        for (int j = threadIdx.x; j < ngt; j += blockDim.x)
            if (s_max[j] > 0) atomicMax(&p.gmax[(size_t)b * G + j], s_max[j]);
    } else {
        const int total = __reduce_add_sync(0xffffffffu, my_pos);
        if ((threadIdx.x & 31) == 0 && total) atomicAdd(&p.npos[b], total);
    }
}

// ---------------------------------------------------------------------------------------------------- losses
// sigmoid_focal_loss (losses.py:31-52), gamma 2, alpha 0.25, one element: bce_with_logits * weight * pt^2.
__device__ __forceinline__ float focal_term(float x, float t, float w) {
    const float p = 1.f / (1.f + expf(-x));
    const float pt = __fadd_rn(__fmul_rn(1.f - p, t), __fmul_rn(p, 1.f - t));
    float wt = __fmul_rn(__fadd_rn(__fmul_rn(0.25f, t), __fmul_rn(0.75f, 1.f - t)), w);
    wt = __fmul_rn(wt, __fmul_rn(pt, pt));
    const float bce = fmaxf(x, 0.f) - x * t + log1pf(expf(-fabsf(x)));
    return __fmul_rn(bce, wt);
}

// smooth_l1_loss (losses.py:69-81), beta 1/9 (an fp32 scalar, as torch casts it).
__device__ __forceinline__ float smooth_l1(float p, float t) {
    const float beta = (float)(1.0 / 9.0), half_beta = (float)(0.5 / 9.0);
    const float d = fabsf(__fsub_rn(p, t));
    return d < beta ? __fdiv_rn(__fmul_rn(__fmul_rn(0.5f, d), d), beta) : __fsub_rn(d, half_beta);
}

// F.cross_entropy of two logits.
__device__ __forceinline__ float ce2(float l0, float l1, int label) {
    const float m = fmaxf(l0, l1);
    const float lse = m + logf(expf(l0 - m) + expf(l1 - m));
    return lse - (label ? l1 : l0);
}

// Sum kSlots fp64 values over the block in a fixed order; thread 0 stores them to part[block][slot].
__device__ __forceinline__ void block_partials(double* acc, double* __restrict__ part) {
    __shared__ double s[kThreads / 32][kSlots];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kSlots; ++k) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) s[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < kSlots) {
        double v = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) v += s[w][threadIdx.x];
        part[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * kSlots + threadIdx.x] = v;
    }
}

struct RpnLossParams {
    const float* head;
    int stride, H, W, ncls, cls_off, dir_off, n;     // n = anchors per frame
    const float* anchors;
    int anchors_per_frame;
    const int* labels;
    const float* targets;
    const int* npos;
};

// SSDRotateHead.loss per anchor (ssd_rotate_head.py:160-216,261-305): NormByNumPositives per frame, sigmoid focal
// classification, smooth-L1 on the sin-difference encoding, direction cross-entropy weighted like the positives.
__global__ void __launch_bounds__(kThreads) rpn_loss_kernel(const RpnLossParams p, double* __restrict__ part) {
    const int b = blockIdx.y;
    const float nf = fmaxf((float)p.npos[b], 1.f);
    double acc[kSlots] = {0.0, 0.0, 0.0, 0.0};      // loc, cls, dir
    const int hw = p.H * p.W;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += gridDim.x * blockDim.x) {
        const size_t o = (size_t)b * p.n + i;
        const int lab = p.labels[o];
        const int rot = i & 1, t = i >> 1, c = t / hw, pix = t - c * hw;
        const float* px = p.head + ((size_t)b * hw + pix) * p.stride;
        const float wc = lab >= 0 ? 1.f / nf : 0.f;
        const float* cl = px + p.cls_off + c * (2 * p.ncls) + rot * p.ncls;
        for (int j = 0; j < p.ncls; ++j) acc[1] += (double)focal_term(cl[j], lab == j + 1 ? 1.f : 0.f, wc);
        if (lab > 0) {
            const float wr = 1.f / nf;
            const float* bp = px + c * 14 + rot * 7;
            const float* tg = p.targets + o * 7;
            double l = 0.0;
            for (int e = 0; e < 6; ++e) l += (double)__fmul_rn(smooth_l1(bp[e], tg[e]), wr);
            const float pe = __fmul_rn(sinf(bp[6]), cosf(tg[6])), te = __fmul_rn(cosf(bp[6]), sinf(tg[6]));
            l += (double)__fmul_rn(smooth_l1(pe, te), wr);
            acc[0] += l;
            const float* a = p.anchors + ((p.anchors_per_frame ? o : (size_t)i) * 7);
            const int dl = __fadd_rn(tg[6], a[6]) > 0.f;
            const float* dp = px + p.dir_off + c * 4 + rot * 2;
            acc[2] += (double)__fmul_rn(ce2(dp[0], dp[1], dl), wr);
        }
    }
    block_partials(acc, part);
}

// PSWarpHead.loss (ssd_rotate_head.py:450-485): focal loss on the scores, weights (pos + neg) over the positives of
// the whole batch.
__global__ void __launch_bounds__(kThreads)
pswarp_loss_kernel(const float* __restrict__ scores, const int* __restrict__ labels, int batch, int n,
                   const int* __restrict__ npos, double* __restrict__ part) {
    int tot = 0;
    for (int b = 0; b < batch; ++b) tot += npos[b];
    const float wn = 1.f / fmaxf((float)tot, 1.f);
    double acc[kSlots] = {0.0, 0.0, 0.0, 0.0};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < batch * n; i += gridDim.x * blockDim.x) {
        const int lab = labels[i];
        if (lab >= 0) acc[0] += (double)focal_term(scores[i], lab > 0 ? 1.f : 0.f, wn);
    }
    block_partials(acc, part);
}

// SpMiddleFHD.aux_loss (cmn.py:72-100): focal loss on point_cls with weight 1 / max(#pos, 1) for every point and
// smooth-L1 on point_reg for the positives with the same normaliser.
__global__ void __launch_bounds__(kThreads)
aux_loss_kernel(const float* __restrict__ cls, const float* __restrict__ reg, const int* __restrict__ labels,
                const float* __restrict__ offsets, const int* __restrict__ d_rows, int rows_cap,
                const int* __restrict__ npos, double* __restrict__ part) {
    const int rows = min(d_rows[0], rows_cap);
    const float wn = 1.f / fmaxf((float)npos[0], 1.f);
    double acc[kSlots] = {0.0, 0.0, 0.0, 0.0};
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
        const int lab = labels[r];
        acc[0] += (double)focal_term(cls[r], lab > 0 ? 1.f : 0.f, wn);
        if (lab > 0)
            for (int e = 0; e < 3; ++e)
                acc[1] += (double)__fmul_rn(smooth_l1(reg[(size_t)r * 3 + e], offsets[(size_t)r * 3 + e]), wn);
    }
    block_partials(acc, part);
}

// One block: out[k] = (float)(sum over blocks of part[.][k]) / divisor * scale[k], summed in block order.
__global__ void __launch_bounds__(kThreads)
final_reduce_kernel(const double* __restrict__ part, int nblocks, int nout, float divisor, float s0, float s1,
                    float s2, float* __restrict__ out) {
    __shared__ double s[kThreads];
    const float scale[3] = {s0, s1, s2};
    for (int k = 0; k < nout; ++k) {
        double v = 0.0;
        for (int i = threadIdx.x; i < nblocks; i += kThreads) v += part[(size_t)i * kSlots + k];
        s[threadIdx.x] = v;
        __syncthreads();
        for (int w = kThreads / 2; w > 0; w >>= 1) {
            if ((int)threadIdx.x < w) s[threadIdx.x] += s[threadIdx.x + w];
            __syncthreads();
        }
        if (threadIdx.x == 0) out[k] = ((float)s[0] / divisor) * scale[k];
        __syncthreads();
    }
}

// CTAs per frame of the loss and assignment kernels; the partial sums' workspace is sized for this bound.
int loss_grid(long long work) { return sassd_grid(work, kThreads, 2); }

__global__ void gt_cap_check_kernel(const int* __restrict__ d_ngt, int batch, int gt_cap, int* __restrict__ status) {
    for (int b = threadIdx.x; b < batch; b += blockDim.x)
        if (d_ngt[b] > gt_cap) atomicOr(status, SASSD_FLAG_GT_CAP);
}

}  // namespace

extern "C" size_t sassd_loss_workspace_bytes(int batch, int gt_cap) {
    const size_t part = (size_t)sassd_num_sms() * 2 * (size_t)(batch > 0 ? batch : 1) * kSlots * sizeof(double);
    const size_t gmax = (size_t)(batch > 0 ? batch : 1) * (gt_cap > 0 ? gt_cap : 1) * sizeof(int);
    return part + ((gmax + 255) / 256) * 256;
}

extern "C" int sassd_points_in_boxes(const float* points_mean, const int32_t* d_rows, int rows_cap, const float* gt,
                                     const int32_t* d_ngt, int batch, int gt_cap, int32_t* labels, float* offsets,
                                     int32_t* d_npos, int32_t* d_status, sassd_stream_t stream) {
    if (!points_mean || !d_rows || !gt || !d_ngt || !labels || !offsets || !d_npos || rows_cap < 1 || batch < 1 ||
        gt_cap < 1 || gt_cap > SASSD_GT_CAP_MAX)
        return SASSD_ERR_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    cudaMemsetAsync(d_npos, 0, sizeof(int), s);
    if (d_status) gt_cap_check_kernel<<<1, 32, 0, s>>>(d_ngt, batch, gt_cap, d_status);
    points_in_boxes_kernel<<<sassd_grid(rows_cap, kThreads, 4), kThreads, 0, s>>>(
        points_mean, d_rows, rows_cap, gt, d_ngt, batch, gt_cap, labels, offsets, d_npos);
    return sassd_check_launch();
}

namespace {
int run_assign(AssignParams& p, cudaStream_t s, int32_t* d_status, void* ws, size_t ws_bytes) {
    const size_t need = sassd_loss_workspace_bytes(p.batch, p.gt_cap);
    if (!ws || ws_bytes < need) return SASSD_ERR_WORKSPACE;
    const size_t part = (size_t)sassd_num_sms() * 2 * (size_t)p.batch * kSlots * sizeof(double);
    p.gmax = (int*)((char*)ws + part);
    cudaMemsetAsync(p.gmax, 0, (size_t)p.batch * p.gt_cap * sizeof(int), s);
    cudaMemsetAsync(p.npos, 0, (size_t)p.batch * sizeof(int), s);
    if (d_status) gt_cap_check_kernel<<<1, 32, 0, s>>>(p.d_ngt, p.batch, p.gt_cap, d_status);
    const size_t smem = (size_t)p.gt_cap * (7 + 5) * sizeof(float) + (size_t)p.gt_cap * 3 * sizeof(int);
    dim3 grid(loss_grid(p.n), p.batch);
    assign_kernel<<<grid, kThreads, smem, s>>>(p, 0);
    assign_kernel<<<grid, kThreads, smem, s>>>(p, 1);
    return sassd_check_launch();
}
}  // namespace

extern "C" int sassd_assign_rpn(const float* anchors, int anchors_per_frame, const uint8_t* mask, int n_anchors,
                                int num_class, const float* gt, const int32_t* gt_class, const int32_t* gt_label,
                                const int32_t* d_ngt, int batch, int gt_cap, const float* host_pos_thr,
                                const float* host_neg_thr, int32_t* labels, float* targets, float* ious,
                                int32_t* d_npos, int32_t* d_status, void* ws, size_t ws_bytes,
                                sassd_stream_t stream) {
    if (!anchors || !mask || !gt || !gt_class || !gt_label || !d_ngt || !host_pos_thr || !host_neg_thr || !labels ||
        !d_npos || batch < 1 || gt_cap < 1 || gt_cap > SASSD_GT_CAP_MAX || num_class < 1 ||
        num_class > kMaxClasses || n_anchors < 1 || n_anchors % num_class)
        return SASSD_ERR_ARG;
    AssignParams p = {};
    p.mode = 0;
    p.batch = batch; p.gt_cap = gt_cap; p.n = n_anchors;
    p.gt = gt; p.gt_class = gt_class; p.gt_label = gt_label; p.d_ngt = d_ngt;
    p.anchors = anchors; p.anchors_per_frame = anchors_per_frame ? 1 : 0; p.num_class = num_class;
    p.per_class = n_anchors / num_class; p.mask = mask;
    for (int c = 0; c < num_class; ++c) { p.pos_thr[c] = host_pos_thr[c]; p.neg_thr[c] = host_neg_thr[c]; }
    p.labels = labels; p.targets = targets; p.ious = ious; p.npos = d_npos;
    return run_assign(p, (cudaStream_t)stream, d_status, ws, ws_bytes);
}

extern "C" int sassd_assign_pswarp(const float* gt, const int32_t* d_ngt, int batch, int gt_cap, const float* boxes,
                                   int n_box, const int32_t* d_head, int head_cap, const int32_t* d_k, float pos_thr,
                                   float neg_thr, int32_t* labels, float* ious, int32_t* d_npos, int32_t* d_status,
                                   void* ws, size_t ws_bytes, sassd_stream_t stream) {
    if (!gt || !d_ngt || !boxes || !d_k || !labels || !d_npos || batch < 1 || gt_cap < 1 ||
        gt_cap > SASSD_GT_CAP_MAX || n_box < 1 || head_cap < 0 || head_cap > n_box || (head_cap > 0 && !d_head))
        return SASSD_ERR_ARG;
    AssignParams p = {};
    p.mode = 1;
    p.batch = batch; p.gt_cap = gt_cap; p.n = n_box;
    p.gt = gt; p.d_ngt = d_ngt;
    p.boxes = boxes; p.d_head = head_cap > 0 ? d_head : nullptr; p.d_k = d_k; p.head_cap = head_cap;
    p.pos_thr[0] = pos_thr; p.neg_thr[0] = neg_thr;
    p.labels = labels; p.ious = ious; p.npos = d_npos;
    return run_assign(p, (cudaStream_t)stream, d_status, ws, ws_bytes);
}

extern "C" int sassd_rpn_loss(const float* head, int head_stride, int batch, int H, int W, int num_class,
                              const float* anchors, int anchors_per_frame, int n_anchors, const int32_t* labels,
                              const float* targets, const int32_t* d_npos, float* out, void* ws, size_t ws_bytes,
                              sassd_stream_t stream) {
    const int na = 2 * num_class;
    if (!head || !anchors || !labels || !targets || !d_npos || !out || batch < 1 || num_class < 1 ||
        n_anchors != num_class * H * W * 2 || head_stride < na * 7 + na * num_class + na * 2)
        return SASSD_ERR_ARG;
    if (!ws || ws_bytes < sassd_loss_workspace_bytes(batch, 1)) return SASSD_ERR_WORKSPACE;
    RpnLossParams p;
    p.head = head; p.stride = head_stride; p.H = H; p.W = W; p.ncls = num_class;
    p.cls_off = na * 7; p.dir_off = na * 7 + na * num_class; p.n = n_anchors;
    p.anchors = anchors; p.anchors_per_frame = anchors_per_frame ? 1 : 0;
    p.labels = labels; p.targets = targets; p.npos = d_npos;
    cudaStream_t s = (cudaStream_t)stream;
    dim3 grid(loss_grid(n_anchors), batch);
    rpn_loss_kernel<<<grid, kThreads, 0, s>>>(p, (double*)ws);
    // rpn_loc_loss = loc / B * 2, rpn_cls_loss = cls / B, rpn_dir_loss = dir / B * 0.2 (ssd_rotate_head.py:289-303)
    final_reduce_kernel<<<1, kThreads, 0, s>>>((const double*)ws, grid.x * grid.y, 3, (float)batch, 2.f, 1.f, .2f,
                                               out);
    return sassd_check_launch();
}

extern "C" int sassd_pswarp_loss(const float* scores, const int32_t* labels, int batch, int n_box,
                                 const int32_t* d_npos, float* out, void* ws, size_t ws_bytes,
                                 sassd_stream_t stream) {
    if (!scores || !labels || !d_npos || !out || batch < 1 || n_box < 1) return SASSD_ERR_ARG;
    if (!ws || ws_bytes < sassd_loss_workspace_bytes(batch, 1)) return SASSD_ERR_WORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = loss_grid((long long)batch * n_box);
    pswarp_loss_kernel<<<grid, kThreads, 0, s>>>(scores, labels, batch, n_box, d_npos, (double*)ws);
    final_reduce_kernel<<<1, kThreads, 0, s>>>((const double*)ws, grid, 1, (float)batch, 1.f, 1.f, 1.f, out);
    return sassd_check_launch();
}

extern "C" int sassd_aux_loss(const float* point_cls, const float* point_reg, const int32_t* labels,
                              const float* offsets, const int32_t* d_rows, int rows_cap, int batch,
                              const int32_t* d_npos, float* out, void* ws, size_t ws_bytes, sassd_stream_t stream) {
    if (!point_cls || !point_reg || !labels || !offsets || !d_rows || !d_npos || !out || rows_cap < 1 || batch < 1)
        return SASSD_ERR_ARG;
    if (!ws || ws_bytes < sassd_loss_workspace_bytes(batch, 1)) return SASSD_ERR_WORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = loss_grid(rows_cap);
    aux_loss_kernel<<<grid, kThreads, 0, s>>>(point_cls, point_reg, labels, offsets, d_rows, rows_cap, d_npos,
                                              (double*)ws);
    // aux_loss_cls, aux_loss_reg, each divided by the number of frames (cmn.py:93-97)
    final_reduce_kernel<<<1, kThreads, 0, s>>>((const double*)ws, grid, 2, (float)batch, 1.f, 1.f, 1.f, out);
    return sassd_check_launch();
}

// Training-time augmentation of labelled frames: the device side of the reference's PointAugmentor
// (mmdet/core/point_cloud/point_augmentor.py) as prepare_train_img applies it (mmdet/datasets/kitti.py:181-209).
// The host makes every random draw and the per-box geometry (augment.py); these kernels do the per-point work and the
// collision-free noise search.  The scene crop by the sampled boxes is a crop_kernel instance (frustum.cu,
// sassd_augment_drop_points).
//
// Rounding.  The reference runs numba-compiled float32 code and numpy's float32 matmul.  Every product below that the
// reference rounds on its own is __fmul_rn, every sum __fadd_rn, and the 2x2 / 3x3 row-vector rotations are the
// sequential FMA chains numpy and numba's BLAS compute: out_k = fma(z, R2k, fma(y, R1k, fma(x, R0k, +0))).  A float32
// value plus a float64 one (numba's `f32_array += f64_array`, numpy's `f32 += f64 box centre`) is
// (float)((double)a + b).  nvcc contraction never decides a rounding here.
#include "common.cuh"

#define AUG_TRIES_MAX 128
#define AUG_NS_THREADS 256
#define AUG_THREADS 256
#define AUG_MAX_BATCH 256
static_assert(AUG_NS_THREADS % AUG_TRIES_MAX == 0, "whole groups of tries per CTA");

__device__ __forceinline__ float aug_min(float a, float b) { return b < a ? b : a; }    // Python's min / max
__device__ __forceinline__ float aug_max(float a, float b) { return b > a ? b : a; }
__device__ __forceinline__ float aug_addd(float a, double b) {
    return isnan(a) ? __int_as_float(__float_as_int(a) | 0x00400000) : __double2float_rn(__dadd_rn((double)a, b));
}

// (p0*R00 + p1*R10 [+ p2*R20]) as the BLAS chain from +0
__device__ __forceinline__ float aug_dot2(float x, float y, float r0, float r1) {
    return __fmaf_rn(y, r1, __fmaf_rn(x, r0, 0.0f));
}
__device__ __forceinline__ float aug_dot3(float x, float y, float z, float r0, float r1, float r2) {
    return __fmaf_rn(z, r2, __fmaf_rn(y, r1, __fmaf_rn(x, r0, 0.0f)));
}

// BEV standup box (xmin, ymin, xmax, ymax) of 4 corners (corner_to_standup_nd_jit)
__device__ __forceinline__ float4 aug_standup(const float2* c) {
    float4 s = make_float4(c[0].x, c[0].y, c[0].x, c[0].y);
#pragma unroll
    for (int k = 1; k < 4; ++k) {
        s.x = fminf(s.x, c[k].x); s.y = fminf(s.y, c[k].y);
        s.z = fmaxf(s.z, c[k].x); s.w = fmaxf(s.w, c[k].y);
    }
    return s;
}

__device__ __forceinline__ bool aug_ccw_gt(float2 p, float2 q, float2 r) {   // (q.y-p.y)*(r.x-p.x) > (r.y-p.y)*(q.x-p.x)
    return __fmul_rn(__fsub_rn(q.y, p.y), __fsub_rn(r.x, p.x)) > __fmul_rn(__fsub_rn(r.y, p.y), __fsub_rn(q.x, p.x));
}

// every corner of q strictly inside clockwise box a: cross < 0 for each edge
__device__ __forceinline__ bool aug_contains(const float2* a, const float2* q) {
#pragma unroll 1
    for (int l = 0; l < 4; ++l)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 u = a[k], v = a[(k + 1) & 3];
            const float vx = -__fsub_rn(u.x, v.x), vy = -__fsub_rn(u.y, v.y);
            const float cross = __fsub_rn(__fmul_rn(vy, __fsub_rn(u.x, q[l].x)), __fmul_rn(vx, __fsub_rn(u.y, q[l].y)));
            if (cross >= 0.0f) return false;
        }
    return true;
}

// box_collision_test for one pair, with numba-compiled semantics: crossing edges, or either box inside the other
__device__ bool aug_collide(const float2* a, float4 sa, const float2* q, float4 sq) {
    const float iw = __fsub_rn(aug_min(sa.z, sq.z), aug_max(sa.x, sq.x));
    if (!(iw > 0.0f)) return false;
    const float ih = __fsub_rn(aug_min(sa.w, sq.w), aug_max(sa.y, sq.y));
    if (!(ih > 0.0f)) return false;
#pragma unroll 1
    for (int k = 0; k < 4; ++k)
#pragma unroll 1
        for (int l = 0; l < 4; ++l) {
            const float2 A = a[k], B = a[(k + 1) & 3], C = q[l], D = q[(l + 1) & 3];
            if (aug_ccw_gt(A, D, C) != aug_ccw_gt(B, D, C) && aug_ccw_gt(A, C, B) != aug_ccw_gt(A, D, B)) return true;
        }
    return aug_contains(a, q) || aug_contains(q, a);
}

// noise_per_box: one CTA per frame walks its boxes in order.  For box i, thread group g of the tries j tests the try's
// corners against boxes g, g + G, ... (every box's current corners, box i itself excluded); the smallest try with no
// collision is box i's, and its corners replace box i's before box i + 1.  -1: no try succeeded.
__global__ void __launch_bounds__(AUG_NS_THREADS)
aug_noise_kernel(const float* __restrict__ boxes, const float* __restrict__ box_trig, const int* __restrict__ box_off,
                 int tries, const float* __restrict__ try_trig, const double* __restrict__ loc, int* __restrict__ sel,
                 int* __restrict__ status) {
    __shared__ float2 s_c[SASSD_GT_CAP_MAX][4];
    __shared__ float4 s_su[SASSD_GT_CAP_MAX];
    __shared__ int s_coll[AUG_TRIES_MAX];
    __shared__ int s_best;
    const int lo = __ldg(&box_off[blockIdx.x]), total = __ldg(&box_off[blockIdx.x + 1]) - lo;
    const int n = min(total, SASSD_GT_CAP_MAX);
    if (threadIdx.x == 0 && total > SASSD_GT_CAP_MAX) atomicOr(status, SASSD_FLAG_GT_CAP);
    for (int k = n + (int)threadIdx.x; k < total; k += blockDim.x) sel[lo + k] = -1;
    // box2d_to_corner_jit: corners (+-w/2, +-l/2) in the order (-,-), (-,+), (+,+), (+,-), rotated, plus (x, y)
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
        const float* b = boxes + (size_t)(lo + k) * 5;
        const float c = __ldg(&box_trig[2 * (lo + k)]), s = __ldg(&box_trig[2 * (lo + k) + 1]);
        const float hw = __fmul_rn(__ldg(&b[2]), 0.5f), hl = __fmul_rn(__ldg(&b[3]), 0.5f);
        const float lx[4] = {-hw, -hw, hw, hw}, ly[4] = {-hl, hl, hl, -hl};
#pragma unroll
        for (int r = 0; r < 4; ++r)
            s_c[k][r] = make_float2(__fadd_rn(aug_dot2(lx[r], ly[r], c, s), __ldg(&b[0])),
                                    __fadd_rn(aug_dot2(lx[r], ly[r], -s, c), __ldg(&b[1])));
        s_su[k] = aug_standup(s_c[k]);
    }
    const int j = threadIdx.x % AUG_TRIES_MAX, g = threadIdx.x / AUG_TRIES_MAX, G = blockDim.x / AUG_TRIES_MAX;
    for (int i = 0; i < n; ++i) {
        if (g == 0) s_coll[j] = 0;
        if (threadIdx.x == 0) s_best = AUG_TRIES_MAX;
        __syncthreads();
        float2 cc[4];
        if (j < tries) {
            const float bx = __ldg(&boxes[(size_t)(lo + i) * 5]), by = __ldg(&boxes[(size_t)(lo + i) * 5 + 1]);
            const size_t t = (size_t)(lo + i) * tries + j;
            const float c = __ldg(&try_trig[2 * t]), s = __ldg(&try_trig[2 * t + 1]);
            const double ox = __dadd_rn((double)bx, __ldg(&loc[3 * t])), oy = __dadd_rn((double)by, __ldg(&loc[3 * t + 1]));
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const float x = __fsub_rn(s_c[i][r].x, bx), y = __fsub_rn(s_c[i][r].y, by);
                cc[r] = make_float2(aug_addd(aug_dot2(x, y, c, s), ox), aug_addd(aug_dot2(x, y, -s, c), oy));
            }
            const float4 su = aug_standup(cc);
            for (int k = g; k < n; k += G)
                if (k != i && aug_collide(cc, su, s_c[k], s_su[k])) {
                    s_coll[j] = 1;
                    break;
                }
        }
        __syncthreads();
        if (g == 0 && j < tries && !s_coll[j]) atomicMin(&s_best, j);
        __syncthreads();
        const int best = s_best;
        if (threadIdx.x == 0) sel[lo + i] = best < tries ? best : -1;
        if (g == 0 && j == best) {
#pragma unroll
            for (int r = 0; r < 4; ++r) s_c[i][r] = cc[r];
            s_su[i] = aug_standup(cc);
        }
        __syncthreads();
    }
}

extern "C" int sassd_augment_noise_search(const float* boxes, const float* box_trig, const int32_t* d_box_off, int batch,
                                          int tries, const float* try_trig, const double* loc, int32_t* sel,
                                          int32_t* d_status, sassd_stream_t stream) {
    if (!boxes || !box_trig || !d_box_off || !try_trig || !loc || !sel || !d_status) return SASSD_ERR_ARG;
    if (batch < 1 || batch > AUG_MAX_BATCH || tries < 1 || tries > AUG_TRIES_MAX) return SASSD_ERR_ARG;
    aug_noise_kernel<<<batch, AUG_NS_THREADS, 0, (cudaStream_t)stream>>>(boxes, box_trig, d_box_off, tries, try_trig,
                                                                          loc, sel, d_status);
    return sassd_check_launch();
}

// The augmented cloud: per frame, the sampled records' database rows (sample order, each plus its box centre; with
// srec_dz, z then minus srec_dz[s], the box's move onto the frame's road plane, rounded again as numpy's
// `f32_array[:, 2] -= f64` does) and then the scene rows the crop kept.  Each row then takes the transform of the first
// box (in box order) whose fp32 planes contain it (points_transform_: -centre, the noise rotation, +centre, +location
// noise; a box without a successful try rotates by 0), the frame's flip of y, its global rotation and its scaling.
__global__ void __launch_bounds__(AUG_THREADS)
aug_assemble_kernel(const float4* __restrict__ kept, const int* __restrict__ kept_off, int batch,
                    const int* __restrict__ srow_off, const int* __restrict__ srec_off, int n_rec,
                    const int* __restrict__ srec_db, const double* __restrict__ srec_ctr,
                    const double* __restrict__ srec_dz, const float4* __restrict__ db,
                    const int* __restrict__ box_off, const float* __restrict__ planes, const float* __restrict__ centres,
                    const int* __restrict__ sel, int tries, const float* __restrict__ try_trig,
                    const double* __restrict__ loc, const float* __restrict__ frame_tf, int out_cap,
                    float4* __restrict__ out, int* __restrict__ out_off, int* __restrict__ status) {
    __shared__ int s_off[AUG_MAX_BATCH + 1];
    for (int b = threadIdx.x; b <= batch; b += blockDim.x) s_off[b] = __ldg(&kept_off[b]) + __ldg(&srow_off[b]);
    __syncthreads();
    const int total = s_off[batch];
    if (blockIdx.x == 0) {
        for (int b = threadIdx.x; b <= batch; b += blockDim.x) out_off[b] = s_off[b];
        if (threadIdx.x == 0 && total > out_cap) atomicOr(status, SASSD_FLAG_POINTS_CAP);
    }
    const int rows = min(total, out_cap);
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
        const int b = sassd_frame_of(s_off, batch, r);
        const int q = r - s_off[b], s0 = __ldg(&srow_off[b]), ns = __ldg(&srow_off[b + 1]) - s0;
        float4 p;
        if (q < ns) {
            const int gr = s0 + q, s = sassd_frame_of(srec_off, n_rec, gr);
            p = __ldg(&db[__ldg(&srec_db[s]) + gr - __ldg(&srec_off[s])]);
            p.x = aug_addd(p.x, __ldg(&srec_ctr[3 * s]));
            p.y = aug_addd(p.y, __ldg(&srec_ctr[3 * s + 1]));
            p.z = aug_addd(p.z, __ldg(&srec_ctr[3 * s + 2]));
            if (srec_dz) p.z = aug_addd(p.z, -__ldg(&srec_dz[s]));
        } else {
            p = __ldg(&kept[__ldg(&kept_off[b]) + q - ns]);
        }
        const int k1 = __ldg(&box_off[b + 1]);
        for (int k = __ldg(&box_off[b]); k < k1; ++k) {
            if (!fc_inside(p, planes + (size_t)k * 24)) continue;
            const int j = __ldg(&sel[k]);
            float c = 1.0f, sn = 0.0f;
            double l0 = 0.0, l1 = 0.0, l2 = 0.0;
            if (j >= 0) {
                const size_t t = (size_t)k * tries + j;
                c = __ldg(&try_trig[2 * t]);
                sn = __ldg(&try_trig[2 * t + 1]);
                l0 = __ldg(&loc[3 * t]); l1 = __ldg(&loc[3 * t + 1]); l2 = __ldg(&loc[3 * t + 2]);
            }
            const float cx = __ldg(&centres[3 * k]), cy = __ldg(&centres[3 * k + 1]), cz = __ldg(&centres[3 * k + 2]);
            const float x = __fsub_rn(p.x, cx), y = __fsub_rn(p.y, cy), z = __fsub_rn(p.z, cz);
            p.x = aug_addd(__fadd_rn(aug_dot3(x, y, z, c, sn, 0.0f), cx), l0);
            p.y = aug_addd(__fadd_rn(aug_dot3(x, y, z, -sn, c, 0.0f), cy), l1);
            p.z = aug_addd(__fadd_rn(aug_dot3(x, y, z, 0.0f, 0.0f, 1.0f), cz), l2);
            break;
        }
        const float* f = frame_tf + (size_t)b * 6;    // flip, R00, R01, R10, R11, scale
        if (__ldg(&f[0]) != 0.0f) p.y = __int_as_float(__float_as_int(p.y) ^ 0x80000000);
        const float r00 = __ldg(&f[1]), r01 = __ldg(&f[2]), r10 = __ldg(&f[3]), r11 = __ldg(&f[4]), sc = __ldg(&f[5]);
        const float x = aug_dot3(p.x, p.y, p.z, r00, r10, 0.0f), y = aug_dot3(p.x, p.y, p.z, r01, r11, 0.0f),
                    z = aug_dot3(p.x, p.y, p.z, 0.0f, 0.0f, 1.0f);
        out[r] = make_float4(__fmul_rn(x, sc), __fmul_rn(y, sc), __fmul_rn(z, sc), p.w);
    }
}

extern "C" int sassd_augment_assemble(const float* kept, const int32_t* d_kept_off, int batch, const int32_t* d_srow_off,
                                      const int32_t* d_srec_off, int n_rec, const int32_t* d_srec_db,
                                      const double* srec_ctr, const double* srec_dz, const float* db,
                                      const int32_t* d_box_off,
                                      const float* planes, const float* centres, const int32_t* sel, int tries,
                                      const float* try_trig, const double* loc, const float* frame_tf, int out_cap,
                                      float* points_out, int32_t* d_pt_off_out, int32_t* d_status,
                                      sassd_stream_t stream) {
    if (!kept || !d_kept_off || !d_srow_off || !d_srec_off || !d_box_off || !sel || !try_trig || !loc || !frame_tf ||
        !points_out || !d_pt_off_out || !d_status)
        return SASSD_ERR_ARG;
    if (batch < 1 || batch > AUG_MAX_BATCH || n_rec < 0 || tries < 1 || tries > AUG_TRIES_MAX || out_cap < 0)
        return SASSD_ERR_ARG;
    if (n_rec > 0 && (!d_srec_db || !srec_ctr || !db)) return SASSD_ERR_ARG;
    if (srec_dz && n_rec == 0) return SASSD_ERR_ARG;
    if (points_out == kept) return SASSD_ERR_ARG;
    const int grid = sassd_grid(out_cap, AUG_THREADS, 4);
    aug_assemble_kernel<<<grid, AUG_THREADS, 0, (cudaStream_t)stream>>>(
        (const float4*)kept, d_kept_off, batch, d_srow_off, d_srec_off, n_rec, d_srec_db, srec_ctr, srec_dz,
        (const float4*)db, d_box_off, planes, centres, sel, tries, try_trig, loc, frame_tf, out_cap,
        (float4*)points_out, d_pt_off_out, d_status);
    return sassd_check_launch();
}

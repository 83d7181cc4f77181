// SA-SSD's auxiliary point-wise head (reference mmdet/models/necks/cmn.py:121-135, :175-189) on the device:
// the three nearest voxel centres of every voxel mean at the three backbone levels, inverse-distance interpolation of
// the level features and the three Linear layers point_fc (160 -> 64, no activation), point_cls (64 -> 1) and
// point_reg (64 -> 3).
//
// sassd_three_nn is bit-identical to pointnet2's three_nn_kernel_fast (interpolate_gpu.cu:9-56) run on the reference's
// points_mean and tensor2points centres: the same fp32 distance as that kernel's sm_90a SASS,
// d = fma(dz, dz, fma(dx, dx, dy * dy)) with dx = ux - x, and the same strict-< insertion.  The reference scans every known row and skips those of other frames;
// level rows are sorted by flattened (b, z, y, x), so a frame's rows are one contiguous range and only that range is
// scanned here.  Strict < over rows in increasing order keeps the three smallest (d, row) pairs in lexicographic order,
// so the scan can be split over SPLIT lanes per point, each keeping the lexicographic top 3 of its own rows, and merged
// by the same order.  The reference's bests are doubles initialised to 1e40: any finite fp32 d is below both 1e40 and
// +inf, so fp32 bests initialised to +inf decide every comparison the same way, and an empty slot ends as
// (idx 0, dist2 (float)1e40 = +inf).
//
// sassd_point_aux_head computes the weights (sqrt, 1 / (dist + 1e-8), normalised by their sum), the interpolation in
// the reference's order (fma(w2, p2, fma(w1, p1, w0 * p0)), interpolate_gpu.cu:80-102) and the Linear layers in fp32.
//
// Both kernels read the row counts on the device, launch fixed grids, allocate nothing and never synchronise with the
// host: graph-capturable.
#include <cuda_fp16.h>

#include "common.cuh"

// tensor2points (mmdet/core/bbox/transforms.py:218-223) as cmn.py:122-129 calls it: offset (0, -40, -3) and the
// voxel sizes of the three levels are literals in the reference, not read from the config, and so they are here.
__constant__ float c_level_vs[3][3] = {{0.1f, 0.1f, 0.2f}, {0.2f, 0.2f, 0.4f}, {0.4f, 0.4f, 0.8f}};
__constant__ float c_offset[3] = {0.0f, -40.0f, -3.0f};

#define NN_POINTS 64                        // level-0 rows per CTA
#define NN_SPLIT 4                          // lanes that share one point, each scanning every NN_SPLIT-th centre
#define NN_THREADS (NN_POINTS * NN_SPLIT)
#define NN_CHUNK 2048                       // centres staged in shared memory per pass (32 KB)

struct Best3 {
    float d0, d1, d2;
    int i0, i1, i2;
};

// the reference's insertion (strict <): called with rows in increasing order it keeps the lexicographic top 3
__device__ __forceinline__ void nn_insert(Best3& b, float d, int k) {
    if (d < b.d2) {
        if (d < b.d1) {
            b.d2 = b.d1; b.i2 = b.i1;
            if (d < b.d0) {
                b.d1 = b.d0; b.i1 = b.i0;
                b.d0 = d; b.i0 = k;
            } else {
                b.d1 = d; b.i1 = k;
            }
        } else {
            b.d2 = d; b.i2 = k;
        }
    }
}

// (d, k) < (e, j) lexicographically; empty slots are (+inf, -1) and only ever tie with each other
__device__ __forceinline__ bool nn_less(float d, int k, float e, int j) { return d < e || (d == e && k < j); }

__device__ __forceinline__ void nn_insert_lex(Best3& b, float d, int k) {
    if (!nn_less(d, k, b.d2, b.i2)) return;
    if (nn_less(d, k, b.d1, b.i1)) {
        b.d2 = b.d1; b.i2 = b.i1;
        if (nn_less(d, k, b.d0, b.i0)) {
            b.d1 = b.d0; b.i1 = b.i0;
            b.d0 = d; b.i0 = k;
        } else {
            b.d1 = d; b.i1 = k;
        }
    } else {
        b.d2 = d; b.i2 = k;
    }
}

// first row in [0, n) whose batch column is >= b (rows sorted by batch)
__device__ __forceinline__ int nn_lower_bound(const int32_t* __restrict__ coors, int n, int b) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (coors[(size_t)mid * 4] < b) lo = mid + 1; else hi = mid;
    }
    return lo;
}

struct NNLevels {
    const int32_t* coors[3];
    const int32_t* d_rows[3];
};

__global__ void __launch_bounds__(NN_THREADS)
three_nn_kernel(const float* __restrict__ mean, const int32_t* __restrict__ coors0, const int32_t* __restrict__ d_rows0,
                NNLevels lv, int32_t* __restrict__ idx_out, float* __restrict__ dist2_out,
                float* __restrict__ points_mean) {
    __shared__ float4 s_ctr[NN_CHUNK];
    __shared__ int s_range[2];
    const int level = blockIdx.y;
    const int n0 = *d_rows0;
    const int first = blockIdx.x * NN_POINTS;
    if (first >= n0) return;
    const int last = min(first + NN_POINTS, n0) - 1;
    const int p = first + (int)threadIdx.x / NN_SPLIT;
    const int s = (int)threadIdx.x % NN_SPLIT;
    const bool valid = p <= last;
    float ux = 0.f, uy = 0.f, uz = 0.f;
    int fb = -1;
    if (valid) {
        const float4 m = *reinterpret_cast<const float4*>(mean + (size_t)p * 4);
        ux = m.x; uy = m.y; uz = m.z;
        fb = coors0[(size_t)p * 4];
        if (points_mean != nullptr && level == 0 && s == 0)
            *reinterpret_cast<float4*>(points_mean + (size_t)p * 4) = make_float4((float)fb, ux, uy, uz);
    }
    // select by value: indexing the parameter struct with a runtime level would copy it to the stack
    const int32_t* __restrict__ kc = level == 0 ? lv.coors[0] : level == 1 ? lv.coors[1] : lv.coors[2];
    const int nk = *(level == 0 ? lv.d_rows[0] : level == 1 ? lv.d_rows[1] : lv.d_rows[2]);
    const float vx = c_level_vs[level][0], vy = c_level_vs[level][1], vz = c_level_vs[level][2];
    const float hx = __fmul_rn(0.5f, vx), hy = __fmul_rn(0.5f, vy), hz = __fmul_rn(0.5f, vz);
    Best3 b{INFINITY, INFINITY, INFINITY, -1, -1, -1};

    // the tile's rows belong to frames coors0[first] .. coors0[last] (frames are contiguous in row order)
    const int f_first = coors0[(size_t)first * 4], f_last = coors0[(size_t)last * 4];
    for (int f = f_first; f <= f_last; ++f) {
        __syncthreads();                                   // s_range / s_ctr of the previous frame are consumed
        if (threadIdx.x == 0) {
            s_range[0] = nn_lower_bound(kc, nk, f);
            s_range[1] = nn_lower_bound(kc, nk, f + 1);
        }
        __syncthreads();
        const int k0 = s_range[0], k1 = s_range[1];
        const bool mine = valid && fb == f;
        for (int c0 = k0; c0 < k1; c0 += NN_CHUNK) {
            const int cn = min(NN_CHUNK, k1 - c0);
            if (c0 != k0) __syncthreads();
            for (int j = threadIdx.x; j < cn; j += NN_THREADS) {
                const int4 q = *reinterpret_cast<const int4*>(kc + (size_t)(c0 + j) * 4);    // (b, z, y, x)
                // ((idx * vs) + offset) + 0.5 * vs, each operation rounded (tensor2points)
                s_ctr[j] = make_float4(__fadd_rn(__fadd_rn(__fmul_rn((float)q.w, vx), c_offset[0]), hx),
                                       __fadd_rn(__fadd_rn(__fmul_rn((float)q.z, vy), c_offset[1]), hy),
                                       __fadd_rn(__fadd_rn(__fmul_rn((float)q.y, vz), c_offset[2]), hz), 0.f);
            }
            __syncthreads();
            if (mine) {
#pragma unroll 4
                for (int j = s; j < cn; j += NN_SPLIT) {
                    const float4 c = s_ctr[j];
                    const float dx = __fsub_rn(ux, c.x), dy = __fsub_rn(uy, c.y), dz = __fsub_rn(uz, c.z);
                    const float d = __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
                    nn_insert(b, d, c0 + j);
                }
            }
        }
    }
    // merge the NN_SPLIT partial lists of a point (adjacent lanes) in lexicographic (d, row) order
#pragma unroll
    for (int m = 1; m < NN_SPLIT; m <<= 1) {
        const float e0 = __shfl_xor_sync(0xffffffffu, b.d0, m), e1 = __shfl_xor_sync(0xffffffffu, b.d1, m),
                    e2 = __shfl_xor_sync(0xffffffffu, b.d2, m);
        const int j0 = __shfl_xor_sync(0xffffffffu, b.i0, m), j1 = __shfl_xor_sync(0xffffffffu, b.i1, m),
                  j2 = __shfl_xor_sync(0xffffffffu, b.i2, m);
        nn_insert_lex(b, e0, j0);
        nn_insert_lex(b, e1, j1);
        nn_insert_lex(b, e2, j2);
    }
    if (valid && s == 0) {
        const size_t o = ((size_t)p * 3 + level) * 3;
        idx_out[o] = max(b.i0, 0); idx_out[o + 1] = max(b.i1, 0); idx_out[o + 2] = max(b.i2, 0);
        dist2_out[o] = b.d0; dist2_out[o + 1] = b.d1; dist2_out[o + 2] = b.d2;
    }
}

extern "C" int sassd_three_nn(const float* mean, const int32_t* coors0, const int32_t* d_rows0, int rows_cap0,
                              const int32_t* coors1, const int32_t* d_rows1, const int32_t* coors2,
                              const int32_t* d_rows2, const int32_t* coors3, const int32_t* d_rows3, int32_t* idx,
                              float* dist2, float* points_mean, sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!mean || !coors0 || !d_rows0 || !coors1 || !d_rows1 || !coors2 || !d_rows2 || !coors3 || !d_rows3 || !idx ||
        !dist2)
        return SASSD_ERR_ARG;
    if (rows_cap0 < 1) return SASSD_ERR_ARG;
    NNLevels lv{{coors1, coors2, coors3}, {d_rows1, d_rows2, d_rows3}};
    dim3 grid(sassd_div_up(rows_cap0, NN_POINTS), 3);
    three_nn_kernel<<<grid, NN_THREADS, 0, stream>>>(mean, coors0, d_rows0, lv, idx, dist2, points_mean);
    return sassd_check_launch();
}

// ---------------------------------------------------------------------------------------------------------------------
#define AH_THREADS 256
#define AH_WARPS (AH_THREADS / 32)
#define AH_IN 160                            // 32 + 64 + 64 interpolated channels
#define AH_HID 64

struct AHLevels {
    const void* rows[3];
    long long plane_stride[3];               // elements from the hi to the lo plane of split rows
    int row_stride[3];
    int split[3];
};

__constant__ int c_ah_ch[3] = {32, 64, 64};
__constant__ int c_ah_base[3] = {0, 32, 96};

__device__ __forceinline__ float ah_feature(const AHLevels& lv, int l, int row, int c) {
    if (lv.split[l]) {       // x = hi + lo * 2^-11, as split_rows_float / features_cap decode it
        const __half* h = static_cast<const __half*>(lv.rows[l]) + (size_t)row * lv.row_stride[l] + c;
        return __fadd_rn(__half2float(h[0]), __fmul_rn(__half2float(h[lv.plane_stride[l]]), 1.0f / 2048.0f));
    }
    return static_cast<const float*>(lv.rows[l])[(size_t)row * lv.row_stride[l] + c];
}

__global__ void __launch_bounds__(AH_THREADS)
point_aux_head_kernel(const int32_t* __restrict__ idx, const float* __restrict__ dist2,
                      const int32_t* __restrict__ d_rows0, AHLevels lv, const float* __restrict__ w_fc_t,
                      const float* __restrict__ w_out, float* __restrict__ cls, float* __restrict__ reg) {
    __shared__ float s_fc[AH_IN * AH_HID];            // point_fc.weight^T: [in][out]
    __shared__ float s_out[4 * AH_HID];               // point_cls.weight, then point_reg.weight
    __shared__ float s_feat[AH_WARPS][AH_IN];
    for (int i = threadIdx.x; i < AH_IN * AH_HID; i += AH_THREADS) s_fc[i] = w_fc_t[i];
    for (int i = threadIdx.x; i < 4 * AH_HID; i += AH_THREADS) s_out[i] = w_out[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n0 = *d_rows0;
    float* feat = s_feat[warp];
    for (int p = blockIdx.x * AH_WARPS + warp; p < n0; p += gridDim.x * AH_WARPS) {
#pragma unroll
        for (int l = 0; l < 3; ++l) {
            const size_t o = ((size_t)p * 3 + l) * 3;
            float r[3];
            int k[3];
#pragma unroll
            for (int t = 0; t < 3; ++t) {
                k[t] = idx[o + t];
                // pointnet2_utils.py:31 and cmn.py:184-186: dist = sqrt(dist2), 1 / (dist + 1e-8); an empty slot
                // (dist2 = +inf) gets weight 0
                r[t] = __frcp_rn(__fadd_rn(__fsqrt_rn(dist2[o + t]), 1e-8f));
            }
            const float norm = __fadd_rn(__fadd_rn(r[0], r[1]), r[2]);
            const float w0 = __fdiv_rn(r[0], norm), w1 = __fdiv_rn(r[1], norm), w2 = __fdiv_rn(r[2], norm);
            for (int c = lane; c < c_ah_ch[l]; c += 32) {
                const float p0 = ah_feature(lv, l, k[0], c), p1 = ah_feature(lv, l, k[1], c),
                            p2 = ah_feature(lv, l, k[2], c);
                feat[c_ah_base[l] + c] = __fmaf_rn(w2, p2, __fmaf_rn(w1, p1, __fmul_rn(w0, p0)));
            }
        }
        __syncwarp();
        float h0 = 0.f, h1 = 0.f;                     // hidden units lane and lane + 32
#pragma unroll 8
        for (int i = 0; i < AH_IN; ++i) {
            const float x = feat[i];
            h0 = __fmaf_rn(s_fc[i * AH_HID + lane], x, h0);
            h1 = __fmaf_rn(s_fc[i * AH_HID + lane + 32], x, h1);
        }
        float acc[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] = __fmaf_rn(s_out[j * AH_HID + lane + 32], h1, __fmul_rn(s_out[j * AH_HID + lane], h0));
#pragma unroll
        for (int m = 16; m >= 1; m >>= 1)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[j] = __fadd_rn(acc[j], __shfl_xor_sync(0xffffffffu, acc[j], m));
        if (lane == 0) {
            cls[p] = acc[0];
            reg[(size_t)p * 3] = acc[1]; reg[(size_t)p * 3 + 1] = acc[2]; reg[(size_t)p * 3 + 2] = acc[3];
        }
        __syncwarp();                                 // feat is rewritten by the next point
    }
}

extern "C" int sassd_point_aux_head(const int32_t* idx, const float* dist2, const int32_t* d_rows0, int rows_cap0,
                                    const sassd_point_levels* host_levels, const float* w_fc_t, const float* w_out,
                                    float* cls, float* reg, sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!idx || !dist2 || !d_rows0 || !host_levels || !w_fc_t || !w_out || !cls || !reg || rows_cap0 < 1)
        return SASSD_ERR_ARG;
    AHLevels lv;
    static const int ch[3] = {32, 64, 64};
    for (int l = 0; l < 3; ++l) {
        const sassd_point_levels& h = host_levels[l];
        if (!h.rows) return SASSD_ERR_ARG;
        if (h.channels != ch[l] || h.row_stride < h.channels || (h.split && h.plane_stride <= 0))
            return SASSD_ERR_UNSUPPORTED;
        lv.rows[l] = h.rows;
        lv.plane_stride[l] = h.plane_stride;
        lv.row_stride[l] = h.row_stride;
        lv.split[l] = h.split ? 1 : 0;
    }
    const int grid = sassd_grid((long long)rows_cap0, AH_WARPS, 2);
    point_aux_head_kernel<<<grid, AH_THREADS, 0, stream>>>(idx, dist2, d_rows0, lv, w_fc_t, w_out, cls, reg);
    return sassd_check_launch();
}

// KITTI result formatting on the device: results.kitti_bbox2results (reference mmdet/core/bbox/transforms.py:225-279)
// for a whole batch, run on the NMS output (sassd_rescore_nms) inside the captured step.
//
// Per box, every operation mirrors the host formatter's numpy dtype:
//   * ry = limit_period(ry, 0.5, 2*pi) in fp32: ry - floor(ry / P + 0.5) * P with P = (float)(2*pi), each operation
//     rounded on its own (__fdiv_rn / __fadd_rn / __fmul_rn, no contraction);
//   * location = (((x, y, z, 1) @ Tr_velo_to_cam^T) @ R0_rect^T) in fp64, rounded to fp32 (boxes_cam is fp32);
//   * the 8 corners of the camera box (origin (0.5, 1, 0.5), rotation about the camera y axis) in fp32 with sinf / cosf;
//   * their projection (x, y, z, 1) @ P2^T, the division by depth and the min / max in fp64;
//   * alpha = -atan2f(-y, x) + ry in fp32.
// The host's float32 sin / cos / atan2 (numpy's own routines), its einsum for the corner rotation (SIMD, possibly fused)
// and OpenBLAS's dgemm summation order are not CUDA's, so the rows are not bit-identical to kitti_bbox2results.  They
// agree within the bounds tests/test_kitti_format.py states: location and rotation_y within 1 fp32 ulp, alpha within
// 1e-6 rad, the 2-D box within 1e-3 px; dimensions, score and label are copies and match exactly.
//
// A box whose projection lies wholly outside the image (x1 > w, y1 > h, x2 < 0 or y2 < 0) is dropped; the others are
// clipped to [0, w] x [0, h] (np.minimum / np.maximum: a NaN stays NaN).  Kept rows are compacted in detection order.
//
// One CTA per frame, one box per thread and pass: a warp ballot of the keep flags, a prefix over the warps' counts, a
// running base across passes.  No host synchronisation and no status flag: graph-capturable.
#include "common.cuh"

#define KF_THREADS 256
#define KF_WARPS (KF_THREADS / 32)

__global__ void __launch_bounds__(KF_THREADS)
kitti_format_kernel(const float* __restrict__ det, const int* __restrict__ d_ndet, int det_cap,
                    const double* __restrict__ meta, double* __restrict__ rows, int* __restrict__ n_out) {
    __shared__ double s_meta[SASSD_KITTI_META];
    __shared__ int s_cnt[KF_WARPS];
    __shared__ int s_base;
    const int f = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < SASSD_KITTI_META) s_meta[threadIdx.x] = meta[(size_t)f * SASSD_KITTI_META + threadIdx.x];
    if (threadIdx.x == 0) s_base = 0;
    __syncthreads();
    const double* P2 = s_meta;          // [3][4]
    const double* V2C = s_meta + 12;    // [3][4]
    const double* R0 = s_meta + 24;     // [3][3]
    const double img_h = s_meta[33], img_w = s_meta[34];
    const int nd = min(max(d_ndet[f], 0), det_cap);
    const float period = 6.28318530717958647692f;      // np.pi * 2 as the fp32 operand numpy uses

    for (int i0 = 0; i0 < nd; i0 += KF_THREADS) {
        const int i = i0 + (int)threadIdx.x;
        bool keep = false;
        double out[SASSD_KITTI_ROW];
        if (i < nd) {
            const float* d = det + ((size_t)f * det_cap + i) * 9;
            const float x = d[0], y = d[1], z = d[2], bw = d[3], bl = d[4], bh = d[5];
            const float ry = __fsub_rn(d[6], __fmul_rn(floorf(__fadd_rn(__fdiv_rn(d[6], period), 0.5f)), period));
            // velo -> ref -> rect, fp64, then rounded to fp32
            const double hv[4] = {(double)x, (double)y, (double)z, 1.0};
            double ref[3], rect[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                double s = __dmul_rn(hv[0], V2C[4 * r]);
#pragma unroll
                for (int c = 1; c < 4; ++c) s = __dadd_rn(s, __dmul_rn(hv[c], V2C[4 * r + c]));
                ref[r] = s;
            }
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                double s = __dmul_rn(ref[0], R0[3 * r]);
#pragma unroll
                for (int c = 1; c < 3; ++c) s = __dadd_rn(s, __dmul_rn(ref[c], R0[3 * r + c]));
                rect[r] = s;
            }
            const float lx = (float)rect[0], ly = (float)rect[1], lz = (float)rect[2];
            // camera box (l, h, w) = lidar (l, h, w) at columns 4, 5, 3
            const float dim[3] = {bl, bh, bw};
            float sn, cs;
            sn = sinf(ry);
            cs = cosf(ry);
            double u0 = 0.0, v0 = 0.0, u1 = 0.0, v1 = 0.0;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                // corner k of the unit box (corners_nd order), minus the origin (0.5, 1, 0.5)
                const int a = k >> 2, b = (k >> 1) & 1, c = (k ^ (k >> 1)) & 1;
                const float cx = __fmul_rn(dim[0], a ? 0.5f : -0.5f);
                const float cy = __fmul_rn(dim[1], b ? 0.0f : -1.0f);
                const float cz = __fmul_rn(dim[2], c ? 0.5f : -0.5f);
                // corners[a,i,:] @ [[c, 0, -s], [0, 1, 0], [s, 0, c]], summed in j order
                const float px = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(cx, cs), __fmul_rn(cy, 0.0f)), __fmul_rn(cz, sn)), lx);
                const float py = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(cx, 0.0f), __fmul_rn(cy, 1.0f)), __fmul_rn(cz, 0.0f)), ly);
                const float pz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(cx, -sn), __fmul_rn(cy, 0.0f)), __fmul_rn(cz, cs)), lz);
                const double hc[4] = {(double)px, (double)py, (double)pz, 1.0};
                double uvw[3];
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    double s = __dmul_rn(hc[0], P2[4 * r]);
#pragma unroll
                    for (int q = 1; q < 4; ++q) s = __dadd_rn(s, __dmul_rn(hc[q], P2[4 * r + q]));
                    uvw[r] = s;
                }
                const double u = __ddiv_rn(uvw[0], uvw[2]), v = __ddiv_rn(uvw[1], uvw[2]);
                if (k == 0) {
                    u0 = u1 = u;
                    v0 = v1 = v;
                } else {     // np.min / np.max: NaN propagates
                    u0 = (u < u0 || isnan(u)) ? u : u0;
                    v0 = (v < v0 || isnan(v)) ? v : v0;
                    u1 = (u > u1 || isnan(u)) ? u : u1;
                    v1 = (v > v1 || isnan(v)) ? v : v1;
                }
            }
            keep = !((u0 > img_w) || (v0 > img_h) || (u1 < 0.0) || (v1 < 0.0));
            const float alpha = __fadd_rn(-atan2f(-y, x), ry);
            out[0] = (double)alpha;
            out[1] = (u0 < 0.0) ? 0.0 : u0;            // np.maximum(x, 0): NaN stays
            out[2] = (v0 < 0.0) ? 0.0 : v0;
            out[3] = (u1 > img_w) ? img_w : u1;         // np.minimum(x, w)
            out[4] = (v1 > img_h) ? img_h : v1;
            out[5] = (double)bl;
            out[6] = (double)bh;
            out[7] = (double)bw;
            out[8] = (double)lx;
            out[9] = (double)ly;
            out[10] = (double)lz;
            out[11] = (double)ry;
            out[12] = (double)d[7];
            out[13] = (double)d[8];
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_cnt[warp] = __popc(bal);
        __syncthreads();
        int before = s_base;
        for (int w = 0; w < warp; ++w) before += s_cnt[w];
        if (keep) {
            double* o = rows + ((size_t)f * det_cap + before + __popc(bal & ((1u << lane) - 1u))) * SASSD_KITTI_ROW;
#pragma unroll
            for (int c = 0; c < SASSD_KITTI_ROW; ++c) o[c] = out[c];
        }
        __syncthreads();                          // every thread has read s_base and s_cnt
        if (threadIdx.x == 0) {
            int t = s_base;
            for (int w = 0; w < KF_WARPS; ++w) t += s_cnt[w];
            s_base = t;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) n_out[f] = s_base;
}

extern "C" int sassd_kitti_format(const float* det, const int32_t* d_ndet, int batch, int det_cap, const double* meta,
                                  double* rows, int32_t* n_out, sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!det || !d_ndet || !meta || !rows || !n_out) return SASSD_ERR_ARG;
    if (batch < 1 || det_cap < 1) return SASSD_ERR_ARG;
    kitti_format_kernel<<<batch, KF_THREADS, 0, stream>>>(det, d_ndet, det_cap, meta, rows, n_out);
    return sassd_check_launch();
}

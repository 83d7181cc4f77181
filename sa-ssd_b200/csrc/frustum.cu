// Crops of full LiDAR sweeps, compacted in point order: the camera-frustum crop is the device side of the reference's
// offline reduced-cloud step (tools/create_data.py:107-140 -> remove_outside_points, mmdet/core/bbox3d/geometry.py:50-61);
// the image-FOV crop is what its raw-drive dataset applies to every sweep (KittiVideo, mmdet/datasets/kitti.py:394 ->
// get_lidar_in_image_fov, mmdet/datasets/kitti_utils.py:252-263).  One compaction kernel, templated on the keep test.
//
// Frustum keep test: points_in_convex_polygon_3d_jit (geometry.py:190-222) for one polygon of 6 faces.  The fp32 coordinates
// are widened to fp64 and s = ((x*n0 + y*n1) + z*n2) + d is evaluated in exactly that order, every operation rounded on
// its own (__dmul_rn / __dadd_rn, no FMA contraction), so the selection is the reference's bit for bit.  `s >= 0`
// rejects, so a NaN coordinate keeps the point, as there.
//
// Image-FOV keep test: the point projected into image 2 through the frame's meta block (results.meta_block: P2,
// Tr_velo_to_cam, R0_rect, img_h, img_w).  x, y, z are widened to fp64; ref = [x,y,z,1] V2C^T, rect = ref R0^T,
// uvw = [rect,1] P2^T, each dot product a sequential FMA chain from k = 0, fma(a3,b3, fma(a2,b2, fma(a1,b1, a0*b0))),
// which is the order numpy's fp64 matmul takes for these shapes (oracle/image_fov.py restates it; the fixture's
// generator checks the two agree on every row).  u = uvw0/uvw2 and v = uvw1/uvw2 are IEEE divisions; the point is kept
// when u < w && u >= 0 && v < h && v >= 0 && x > clip_x, the last comparison in fp32 as numpy makes it on the float32
// cloud.  A NaN coordinate fails every comparison and drops the point; uvw2 <= 0 divides as IEEE says.
//
// One pass over the concatenated frames: FC_CHUNK points per CTA as FC_ROWS rows of FC_THREADS consecutive points
// (one point per thread and row: coalesced 16-byte loads), warp ballots ranked by a scan of the chunk's (row, warp)
// counts, chunk totals chained by decoupled look-back (sassd_lookback, as vox_rank_kernel).  Frames stay concatenated,
// so a kept point's output row is the number of kept points before it in the batch, and d_pt_off_out[b] is the number
// of kept points before d_pt_off[b].  Bound: 16 B read and <= 16 B written per point (HBM bandwidth / latency).
#include "common.cuh"

#define FC_MAX_BATCH 256
#define FC_THREADS 256
#define FC_WARPS (FC_THREADS / 32)
#define FC_ROWS 8
#define FC_CHUNK (FC_THREADS * FC_ROWS)
static_assert(FC_ROWS * FC_WARPS == 64, "the chunk scan gives two (row, warp) counts to each lane of warp 0");

struct FrustumKeep {
    const double* __restrict__ planes;    // [batch][6][4]
    __device__ __forceinline__ bool operator()(float4 p, int frame) const { return fc_inside(p, planes + (size_t)frame * 24); }
};

// a0*b[0] + a1*b[1] + a2*b[2] (+ b[3] when `affine`): a sequential FMA chain from k = 0
template <bool affine>
__device__ __forceinline__ double fov_dot(double a0, double a1, double a2, const double* __restrict__ b) {
    double acc = __fma_rn(a2, __ldg(&b[2]), __fma_rn(a1, __ldg(&b[1]), __dmul_rn(a0, __ldg(&b[0]))));
    if (affine) acc = __fma_rn(1.0, __ldg(&b[3]), acc);
    return acc;
}

struct ImageFovKeep {
    const double* __restrict__ meta;      // [batch][SASSD_KITTI_META]: P2 (12), Tr_velo_to_cam (12), R0_rect (9), h, w
    float clip_x;
    __device__ __forceinline__ bool operator()(float4 p, int frame) const {
        const double* m = meta + (size_t)frame * SASSD_KITTI_META;
        const double x = p.x, y = p.y, z = p.z;
        const double r0 = fov_dot<true>(x, y, z, m + 12), r1 = fov_dot<true>(x, y, z, m + 16),
                     r2 = fov_dot<true>(x, y, z, m + 20);
        const double c0 = fov_dot<false>(r0, r1, r2, m + 24), c1 = fov_dot<false>(r0, r1, r2, m + 27),
                     c2 = fov_dot<false>(r0, r1, r2, m + 30);
        const double w0 = fov_dot<true>(c0, c1, c2, m), w1 = fov_dot<true>(c0, c1, c2, m + 4),
                     w2 = fov_dot<true>(c0, c1, c2, m + 8);
        const double u = __ddiv_rn(w0, w2), v = __ddiv_rn(w1, w2);
        const double h = __ldg(&m[33]), w = __ldg(&m[34]);
        return u < w && u >= 0.0 && v < h && v >= 0.0 && p.x > clip_x;
    }
};

template <class Keep>
__global__ void __launch_bounds__(FC_THREADS)
crop_kernel(const float4* __restrict__ points, const int* __restrict__ pt_off, int n_cap, int batch, Keep inside,
            float4* __restrict__ out, int* __restrict__ off_out, unsigned long long* __restrict__ desc) {
    __shared__ int s_off[FC_MAX_BATCH + 1];
    __shared__ unsigned s_ball[FC_ROWS * FC_WARPS];   // (row, warp) order = point order
    __shared__ int s_ex[FC_ROWS * FC_WARPS];
    __shared__ int s_base, s_total;
    for (int b = threadIdx.x; b <= batch; b += blockDim.x) s_off[b] = min(max(pt_off[b], 0), n_cap);
    __syncthreads();
    const int n = s_off[batch];
    const int c = blockIdx.x;
    const int last = n > 0 ? (n - 1) / FC_CHUNK : 0;    // the chunk that also writes the offsets at the end
    if (c > last) return;
    const int c0 = c * FC_CHUNK;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    float4 p[FC_ROWS];
#pragma unroll
    for (int j = 0; j < FC_ROWS; ++j) {
        const int i = c0 + j * FC_THREADS + (int)threadIdx.x;
        if (i < n) p[j] = __ldg(&points[i]);
    }
    unsigned keep = 0;
#pragma unroll
    for (int j = 0; j < FC_ROWS; ++j) {
        const int i = c0 + j * FC_THREADS + (int)threadIdx.x;
        if (i < n && inside(p[j], sassd_frame_of(s_off, batch, i))) keep |= 1u << j;
    }
#pragma unroll
    for (int j = 0; j < FC_ROWS; ++j) {
        const unsigned bal = __ballot_sync(0xffffffffu, (keep >> j) & 1u);
        if (lane == 0) s_ball[j * FC_WARPS + warp] = bal;
    }
    __syncthreads();
    if (warp == 0) {
        const int a = __popc(s_ball[2 * lane]), b = __popc(s_ball[2 * lane + 1]);
        int inc = a + b;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += t;
        }
        s_ex[2 * lane] = inc - a - b;
        s_ex[2 * lane + 1] = inc - b;
        const int total = __shfl_sync(0xffffffffu, inc, 31);
        volatile unsigned long long* vd = desc;
        if (c > 0 && lane == 0) vd[c] = (SASSD_SCAN_AGG << 32) | (unsigned)total;
        const int base = sassd_lookback(vd, c, lane);
        if (lane == 0) {
            vd[c] = (SASSD_SCAN_PREFIX << 32) | (unsigned)(base + total);
            s_base = base;
            s_total = total;
        }
    }
    __syncthreads();
    const int base = s_base;
    const unsigned lt = (1u << lane) - 1u;
#pragma unroll
    for (int j = 0; j < FC_ROWS; ++j)
        if ((keep >> j) & 1u) {
            const int k = j * FC_WARPS + warp;
            out[base + s_ex[k] + __popc(s_ball[k] & lt)] = p[j];
        }
    // d_pt_off_out[b]: written by the chunk holding input row pt_off[b]; the last chunk also takes the offsets at n
    const int c1 = c0 + FC_CHUNK;
    for (int b = threadIdx.x; b <= batch; b += blockDim.x) {
        const int o = min(s_off[b], n);
        if (o < c0 || (o >= c1 && c != last)) continue;
        int r = s_total;
        if (o < c1) {
            const int q = o - c0, t = q % FC_THREADS;
            const int k = (q / FC_THREADS) * FC_WARPS + (t >> 5);
            r = s_ex[k] + __popc(s_ball[k] & ((1u << (t & 31)) - 1u));
        }
        off_out[b] = base + r;
    }
}

static inline int fc_chunks(int n_points_cap) { return n_points_cap > FC_CHUNK ? sassd_div_up(n_points_cap, FC_CHUNK) : 1; }

extern "C" size_t sassd_frustum_crop_workspace_bytes(int n_points_cap, int batch) {
    (void)batch;   // one look-back descriptor per chunk of the concatenated frames
    return (size_t)fc_chunks(n_points_cap) * sizeof(unsigned long long);
}

// argument checks shared by both crops; then the descriptor reset and the one launch
template <class Keep>
static int crop_launch(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch, const void* params,
                       Keep inside, float* points_out, int32_t* d_pt_off_out, void* ws, size_t ws_bytes,
                       sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!points || !d_pt_off || !params || !points_out || !d_pt_off_out || !ws) return SASSD_ERR_ARG;
    if (batch < 1 || batch > FC_MAX_BATCH || n_points_cap < 0) return SASSD_ERR_ARG;
    if (points == points_out) return SASSD_ERR_ARG;     // a chunk's output rows may hold a later chunk's input rows
    if (ws_bytes < sassd_frustum_crop_workspace_bytes(n_points_cap, batch)) return SASSD_ERR_WORKSPACE;
    const int chunks = fc_chunks(n_points_cap);
    cudaMemsetAsync(ws, 0, (size_t)chunks * sizeof(unsigned long long), stream);   // descriptors: nothing published
    crop_kernel<<<chunks, FC_THREADS, 0, stream>>>((const float4*)points, d_pt_off, n_points_cap, batch, inside,
                                                   (float4*)points_out, d_pt_off_out, (unsigned long long*)ws);
    return sassd_check_launch();
}

extern "C" int sassd_frustum_crop(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch,
                                  const double* planes, float* points_out, int32_t* d_pt_off_out, void* ws,
                                  size_t ws_bytes, sassd_stream_t stream) {
    return crop_launch(points, d_pt_off, n_points_cap, batch, planes, FrustumKeep{planes}, points_out, d_pt_off_out, ws,
                       ws_bytes, stream);
}

extern "C" int sassd_image_fov_crop(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch,
                                    const double* meta, float clip_x, float* points_out, int32_t* d_pt_off_out,
                                    void* ws, size_t ws_bytes, sassd_stream_t stream) {
    return crop_launch(points, d_pt_off, n_points_cap, batch, meta, ImageFovKeep{meta, clip_x}, points_out,
                       d_pt_off_out, ws, ws_bytes, stream);
}

// Keep test of the augmentation's scene crop (the reference's prepare_train_img, mmdet/datasets/kitti.py:187-189): a
// point survives unless it is inside one of its frame's sampled boxes, under the fp32 plane test of float32 boxes.
struct OutsideBoxesKeep {
    const float* __restrict__ planes;     // [total boxes][6][4] fp32
    const int* __restrict__ box_off;      // [batch + 1]: frame b's boxes are [box_off[b], box_off[b + 1])
    __device__ __forceinline__ bool operator()(float4 p, int frame) const {
        const int lo = __ldg(&box_off[frame]), hi = __ldg(&box_off[frame + 1]);
        for (int j = lo; j < hi; ++j)
            if (fc_inside(p, planes + (size_t)j * 24)) return false;
        return true;
    }
};

extern "C" int sassd_augment_drop_points(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch,
                                         const float* planes, const int32_t* d_box_off, float* points_out,
                                         int32_t* d_pt_off_out, void* ws, size_t ws_bytes, sassd_stream_t stream) {
    if (!d_box_off) return SASSD_ERR_ARG;
    return crop_launch(points, d_pt_off, n_points_cap, batch, planes, OutsideBoxesKeep{planes, d_box_off}, points_out,
                       d_pt_off_out, ws, ws_bytes, stream);
}

// ------------------------------------------------------------------------------------------------------------------
// Points in rotated boxes, gathered per box: the reference's ground-truth database step (tools/create_data.py:233-240 ->
// points_in_rbbox, geometry.py:63-74, then gt_points[:, :3] -= box[:3]) and its num_points_in_gt (create_data.py:16-45).
// The membership test is fc_inside, the frustum crop's, applied to each box's 6 planes.
//
// One CTA per (frame, box slot) q = b * box_cap + j scans frame b twice: once to count its members, then - after the
// count's exclusive prefix over q is known from a decoupled look-back (sassd_lookback, one descriptor per q) - to write
// them in input order at seg_off[q] + rank, ranked like crop_kernel's rows.  The second scan stops after the box's last
// member.  A gathered row is (float)((double)p - c) per coordinate, numpy's float32 -= float64; a NaN coordinate keeps
// its bits (quieted), as the host's double round trip does.  Slots j >= nbox[b] count nothing.
__device__ __forceinline__ float rb_shift(float v, double c) {
    return isnan(v) ? __int_as_float(__float_as_int(v) | 0x00400000) : __double2float_rn(__dsub_rn((double)v, c));
}

__global__ void __launch_bounds__(FC_THREADS)
rbbox_gather_kernel(const float4* __restrict__ points, const int* __restrict__ pt_off, int n_cap,
                    const double* __restrict__ planes, const double* __restrict__ centres, const int* __restrict__ nbox,
                    int box_cap, int* __restrict__ counts, int* __restrict__ seg_off, float4* __restrict__ gathered,
                    int gather_cap, int* __restrict__ status, unsigned long long* __restrict__ desc) {
    __shared__ unsigned s_ball[FC_ROWS * FC_WARPS];
    __shared__ int s_ex[FC_ROWS * FC_WARPS];
    __shared__ int s_red[FC_WARPS];
    __shared__ int s_base, s_total, s_chunk;
    const int q = blockIdx.x, b = q / box_cap, j = q - b * box_cap;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int lo = min(max(__ldg(&pt_off[b]), 0), n_cap);
    const int hi = max(min(max(__ldg(&pt_off[b + 1]), 0), n_cap), lo);
    const int nb = __ldg(&nbox[b]);
    if (j == 0 && threadIdx.x == 0 && nb > box_cap) atomicOr(status, SASSD_FLAG_GT_CAP);
    const bool active = j < nb;
    const double* pl = planes + (size_t)q * 24;

    int cnt = 0;
    if (active)
        for (int c0 = lo; c0 < hi; c0 += FC_CHUNK) {
            float4 p[FC_ROWS];
#pragma unroll
            for (int r = 0; r < FC_ROWS; ++r) {
                const int i = c0 + r * FC_THREADS + (int)threadIdx.x;
                if (i < hi) p[r] = __ldg(&points[i]);
            }
#pragma unroll
            for (int r = 0; r < FC_ROWS; ++r)
                if (c0 + r * FC_THREADS + (int)threadIdx.x < hi && fc_inside(p[r], pl)) ++cnt;
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) s_red[warp] = cnt;
    __syncthreads();
    if (warp == 0) {
        int total = lane < FC_WARPS ? s_red[lane] : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
        volatile unsigned long long* vd = desc;
        if (q > 0 && lane == 0) vd[q] = (SASSD_SCAN_AGG << 32) | (unsigned)total;
        const int base = sassd_lookback(vd, q, lane);
        if (lane == 0) {
            vd[q] = (SASSD_SCAN_PREFIX << 32) | (unsigned)(base + total);
            counts[q] = total;
            seg_off[q] = base;
            if (q == (int)gridDim.x - 1) {
                seg_off[q + 1] = base + total;
                if (base + total > gather_cap) atomicOr(status, SASSD_FLAG_GATHER_CAP);
            }
            s_base = base;
            s_total = total;
        }
    }
    __syncthreads();
    const int base = s_base, end = min(base + s_total, gather_cap);
    if (!gathered || base >= end) return;
    const double cx = __ldg(&centres[3 * (size_t)q]), cy = __ldg(&centres[3 * (size_t)q + 1]),
                 cz = __ldg(&centres[3 * (size_t)q + 2]);
    const unsigned lt = (1u << lane) - 1u;
    int run = base;
    for (int c0 = lo; c0 < hi && run < end; c0 += FC_CHUNK) {
        float4 p[FC_ROWS];
        unsigned keep = 0;
#pragma unroll
        for (int r = 0; r < FC_ROWS; ++r) {
            const int i = c0 + r * FC_THREADS + (int)threadIdx.x;
            if (i < hi) p[r] = __ldg(&points[i]);
        }
#pragma unroll
        for (int r = 0; r < FC_ROWS; ++r)
            if (c0 + r * FC_THREADS + (int)threadIdx.x < hi && fc_inside(p[r], pl)) keep |= 1u << r;
#pragma unroll
        for (int r = 0; r < FC_ROWS; ++r) {
            const unsigned bal = __ballot_sync(0xffffffffu, (keep >> r) & 1u);
            if (lane == 0) s_ball[r * FC_WARPS + warp] = bal;
        }
        __syncthreads();
        if (warp == 0) {
            const int a = __popc(s_ball[2 * lane]), c = __popc(s_ball[2 * lane + 1]);
            int inc = a + c;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, inc, d);
                if (lane >= d) inc += t;
            }
            s_ex[2 * lane] = inc - a - c;
            s_ex[2 * lane + 1] = inc - c;
            if (lane == 31) s_chunk = inc;
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < FC_ROWS; ++r)
            if ((keep >> r) & 1u) {
                const int k = r * FC_WARPS + warp;
                const int o = run + s_ex[k] + __popc(s_ball[k] & lt);
                if (o < end) gathered[o] = make_float4(rb_shift(p[r].x, cx), rb_shift(p[r].y, cy), rb_shift(p[r].z, cz), p[r].w);
            }
        run += s_chunk;
        __syncthreads();    // s_ball / s_ex / s_chunk are rewritten by the next chunk
    }
}

extern "C" size_t sassd_points_in_rbboxes_workspace_bytes(int n_points_cap, int batch, int box_cap) {
    (void)n_points_cap;   // one look-back descriptor per (frame, box slot)
    return (size_t)(batch > 0 ? batch : 0) * (size_t)(box_cap > 0 ? box_cap : 0) * sizeof(unsigned long long);
}

extern "C" int sassd_points_in_rbboxes(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch,
                                       const double* planes, const double* centres, const int32_t* d_nbox, int box_cap,
                                       int32_t* counts, int32_t* seg_off, float* gathered, int gather_cap,
                                       int32_t* d_status, void* ws, size_t ws_bytes, sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!points || !d_pt_off || !planes || !centres || !d_nbox || !counts || !seg_off || !d_status || !ws)
        return SASSD_ERR_ARG;
    if (batch < 1 || batch > FC_MAX_BATCH || n_points_cap < 0) return SASSD_ERR_ARG;
    if (box_cap < 1 || box_cap > SASSD_GT_CAP_MAX || gather_cap < 0 || (!gathered && gather_cap > 0))
        return SASSD_ERR_ARG;
    if (gathered == points) return SASSD_ERR_ARG;
    if (ws_bytes < sassd_points_in_rbboxes_workspace_bytes(n_points_cap, batch, box_cap)) return SASSD_ERR_WORKSPACE;
    const int segs = batch * box_cap;
    cudaMemsetAsync(ws, 0, (size_t)segs * sizeof(unsigned long long), stream);   // descriptors: nothing published
    rbbox_gather_kernel<<<segs, FC_THREADS, 0, stream>>>((const float4*)points, d_pt_off, n_points_cap, planes, centres,
                                                         d_nbox, box_cap, counts, seg_off, (float4*)gathered,
                                                         gather_cap, d_status, (unsigned long long*)ws);
    return sassd_check_launch();
}

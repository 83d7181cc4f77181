// Camera-frustum crop of full LiDAR sweeps: the device side of the reference's offline reduced-cloud step
// (tools/create_data.py:107-140 -> remove_outside_points, mmdet/core/bbox3d/geometry.py:50-61).
//
// Keep test: points_in_convex_polygon_3d_jit (geometry.py:190-222) for one polygon of 6 faces.  The fp32 coordinates
// are widened to fp64 and s = ((x*n0 + y*n1) + z*n2) + d is evaluated in exactly that order, every operation rounded on
// its own (__dmul_rn / __dadd_rn, no FMA contraction), so the selection is the reference's bit for bit.  `s >= 0`
// rejects, so a NaN coordinate keeps the point, as there.
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

__device__ __forceinline__ bool fc_inside(float4 p, const double* __restrict__ pl) {
    const double x = p.x, y = p.y, z = p.z;
    bool in = true;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const double s = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, __ldg(&pl[4 * k])), __dmul_rn(y, __ldg(&pl[4 * k + 1]))),
                                             __dmul_rn(z, __ldg(&pl[4 * k + 2]))),
                                   __ldg(&pl[4 * k + 3]));
        in &= !(s >= 0.0);
    }
    return in;
}

__global__ void __launch_bounds__(FC_THREADS)
frustum_crop_kernel(const float4* __restrict__ points, const int* __restrict__ pt_off, int n_cap, int batch,
                    const double* __restrict__ planes, float4* __restrict__ out, int* __restrict__ off_out,
                    unsigned long long* __restrict__ desc) {
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
        if (i < n && fc_inside(p[j], planes + (size_t)sassd_frame_of(s_off, batch, i) * 24)) keep |= 1u << j;
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

extern "C" int sassd_frustum_crop(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch,
                                  const double* planes, float* points_out, int32_t* d_pt_off_out, void* ws,
                                  size_t ws_bytes, sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!points || !d_pt_off || !planes || !points_out || !d_pt_off_out || !ws) return SASSD_ERR_ARG;
    if (batch < 1 || batch > FC_MAX_BATCH || n_points_cap < 0) return SASSD_ERR_ARG;
    if (points == points_out) return SASSD_ERR_ARG;     // a chunk's output rows may hold a later chunk's input rows
    if (ws_bytes < sassd_frustum_crop_workspace_bytes(n_points_cap, batch)) return SASSD_ERR_WORKSPACE;
    const int chunks = fc_chunks(n_points_cap);
    cudaMemsetAsync(ws, 0, (size_t)chunks * sizeof(unsigned long long), stream);   // descriptors: nothing published
    frustum_crop_kernel<<<chunks, FC_THREADS, 0, stream>>>((const float4*)points, d_pt_off, n_points_cap, batch, planes,
                                                           (float4*)points_out, d_pt_off_out, (unsigned long long*)ws);
    return sassd_check_launch();
}

// Deterministic GPU voxelizer + SimpleVoxel mean + anchors_mask.
//
// Reproduces, bit for bit, the sequential reference loop
// (mmdet/ops/points_op/points_ops.py:4-50): voxel ids by first touch, the
// first `max_points` points of every voxel in point order, and the hard stop
// at the first point that would open voxel number `max_voxels`.
//
// Parallel formulation (SURVEY.md §A.1):
//   1. insert : every in-range point hashes its (z,y,x) cell into a per-frame
//               open-addressing table (no 360 MB dense grid as in
//               points_ops.py:145); first[slot] = min point index,
//               and the point is pushed on the slot's lock-free list.
//   2. rank   : one CTA per frame scans the points in order; a point is a
//               voxel "opener" iff first[slot] == its index; voxel id = number
//               of openers before it; the opener with id == max_voxels marks
//               the cut index (every point at or after it is dropped).
//   3. emit   : each opener walks its slot list, keeps the max_points smallest
//               point indices below the cut, and writes voxels / coors /
//               num_points / mean rows at frame_row_offset + voxel id.
// Traffic: 16 B/point read + 116 B/voxel written (+ table, L2-resident).
#include "common.cuh"

#define VOX_MAX_BATCH 256
#define VOX_MAX_PTS 8

struct VoxConst {
    float vs[3], lo[3];
    int grid[3];
    int max_points, max_voxels;
};

__global__ void __launch_bounds__(256)
vox_insert_kernel(const float4* __restrict__ points, const int* __restrict__ pt_off, int batch, VoxConst P,
                  int slots, int* __restrict__ keys, int* __restrict__ first, int* __restrict__ head,
                  int* __restrict__ pt_slot, int* __restrict__ pt_next, int* __restrict__ status,
                  int* __restrict__ frame_m, int* __restrict__ frame_cut, unsigned long long* __restrict__ rank_desc,
                  int n_desc) {
    __shared__ int s_off[VOX_MAX_BATCH + 1];
    for (int b = threadIdx.x; b <= batch; b += blockDim.x) s_off[b] = pt_off[b];
    __syncthreads();
    if (blockIdx.x == 0) {          // presets for vox_rank_kernel (the next launch): no voxel, no cut, nothing published
        for (int b = threadIdx.x; b < batch; b += blockDim.x) { frame_m[b] = 0; frame_cut[b] = s_off[b + 1]; }
        for (int i = threadIdx.x; i < n_desc; i += blockDim.x) rank_desc[i] = 0ull;
    }
    const int n = s_off[batch];
    const uint32_t mask = (uint32_t)slots - 1u;
    const int lane = threadIdx.x & 31;
    // Warp-aggregated insertion: the loop is warp-uniform (a warp owns 32 consecutive points - in a real Velodyne file
    // consecutive returns of a beam mostly share a voxel).  Lanes whose points fall into the same cell of the same
    // frame find each other with __match_any_sync; only the group's lowest lane probes the table (one atomicCAS chain
    // per distinct cell instead of one per point), takes the atomicMin for the group (it holds the smallest index) and
    // the group enters the slot's list as one pre-linked chain with a single atomicExch.
    for (int base_i = blockIdx.x * blockDim.x + (threadIdx.x & ~31); base_i < n; base_i += gridDim.x * blockDim.x) {
        const int i = base_i + lane;
        bool ok = false;
        int b = 0, cell = 0;
        if (i < n) {
            const float4 p = __ldg(&points[i]);
            // fp32 subtract, IEEE divide, floor — exactly numba's float32 arithmetic (points_ops.py:31)
            const float cx = floorf(__fdiv_rn(__fsub_rn(p.x, P.lo[0]), P.vs[0]));
            const float cy = floorf(__fdiv_rn(__fsub_rn(p.y, P.lo[1]), P.vs[1]));
            const float cz = floorf(__fdiv_rn(__fsub_rn(p.z, P.lo[2]), P.vs[2]));
            // (c < 0 || c >= grid) rejects; non-finite coordinates are rejected too (the
            // reference's behaviour is undefined there: NaN passes both tests and is cast to int)
            ok = (cx >= 0.f) && (cx < (float)P.grid[0]) && (cy >= 0.f) && (cy < (float)P.grid[1]) &&
                 (cz >= 0.f) && (cz < (float)P.grid[2]);
            if (ok) {
                b = sassd_frame_of(s_off, batch, i);
                cell = ((int)cz * P.grid[1] + (int)cy) * P.grid[0] + (int)cx;
            }
        }
        int slot = -1;
        const unsigned okmask = __ballot_sync(0xffffffffu, ok);
        if (ok) {
            // a warp's 32 points span at most two frames in practice; the frame goes into the match key's top bits
            const unsigned long long key = ((unsigned long long)(unsigned)b << 32) | (unsigned)cell;
            const unsigned peers = __match_any_sync(okmask, key);
            const int leader = __ffs(peers) - 1;
            if (lane == leader) {
                int* fk = keys + (size_t)b * slots;
                // bounded probe: the table holds >= 2x the frame's points, so this always terminates early
                uint32_t s = sassd_hash32((uint32_t)cell) & mask;
                int probes = 0;
                while (true) {
                    int prev = atomicCAS(&fk[s], SASSD_EMPTY_KEY, cell);
                    if (prev == SASSD_EMPTY_KEY || prev == cell) { slot = b * slots + (int)s; break; }
                    s = (s + 1) & mask;
                    if (++probes >= slots) { atomicOr(status, SASSD_FLAG_HASH_FULL); break; }
                }
                if (slot >= 0) atomicMin(&first[slot], i);       // lowest lane = smallest point index of the group
            }
            slot = __shfl_sync(peers, slot, leader);
            if (slot >= 0) {
                const unsigned higher = peers & ~((2u << lane) - 1u);
                if (higher) pt_next[i] = base_i + (__ffs(higher) - 1);                 // next point of the group
                else pt_next[i] = atomicExch(&head[slot], base_i + leader);           // tail -> old head; head -> group
            }
        }
        if (i < n) pt_slot[i] = slot;
    }
}

// Ordered ranking of voxel openers (a point opens a voxel when it is the first point of its cell): rank = number of
// openers before it in the frame's point order - the reference's first-touch voxel order (points_ops.py:4-50).
// Round 1: one CTA per frame, 32 points per thread in three 32x-unrolled passes - 17-24 us at the very start of every
// step's critical path, most of it instruction fetch for code that runs once.  Now VR_CHUNK points per CTA (8
// consecutive points per thread), the chunk totals chained by decoupled look-back (descriptors zeroed, and frame_m /
// frame_cut preset, by vox_insert_kernel, which runs before).
#define VR_PTS 8
#define VR_CHUNK (1024 * VR_PTS)
__global__ void __launch_bounds__(1024)
vox_rank_kernel(const int* __restrict__ pt_off, const int* __restrict__ pt_slot, const int* __restrict__ first,
                int* __restrict__ vid, int max_voxels, int* __restrict__ frame_m, int* __restrict__ frame_cut,
                unsigned long long* __restrict__ desc, int chunks_max) {
    __shared__ int s_scan[33];
    __shared__ int s_base;
    const int b = blockIdx.y, c = blockIdx.x;
    const int beg = pt_off[b], end = pt_off[b + 1];
    const int nchunks = (end - beg + VR_CHUNK - 1) / VR_CHUNK;
    if (c >= nchunks) return;
    const int t0 = beg + c * VR_CHUNK + (int)threadIdx.x * VR_PTS;
    uint32_t flags = 0;
    int slots_l[VR_PTS];
#pragma unroll
    for (int j = 0; j < VR_PTS; ++j) slots_l[j] = (t0 + j < end) ? __ldg(&pt_slot[t0 + j]) : -1;
#pragma unroll
    for (int j = 0; j < VR_PTS; ++j) {
        const int s = slots_l[j];
        if (s >= 0 && __ldg(&first[s]) == t0 + j) flags |= 1u << j;
    }
    int total;
    const int ex = sassd_block_exscan(__popc(flags), s_scan, &total);
    if (threadIdx.x < 32) {
        volatile unsigned long long* vd = desc + (size_t)b * chunks_max;
        const int lane = threadIdx.x;
        if (c > 0 && lane == 0) vd[c] = (SASSD_SCAN_AGG << 32) | (unsigned)total;
        const int base = sassd_lookback(vd, c, lane);
        if (lane == 0) {
            vd[c] = (SASSD_SCAN_PREFIX << 32) | (unsigned)(base + total);
            s_base = base;
            if (c == nchunks - 1) frame_m[b] = min(base + total, max_voxels);
        }
    }
    __syncthreads();
    int rank = s_base + ex;
#pragma unroll
    for (int j = 0; j < VR_PTS; ++j) {
        if (flags & (1u << j)) {
            vid[slots_l[j]] = rank < max_voxels ? rank : -1;
            if (rank == max_voxels) frame_cut[b] = t0 + j;       // the first opener past the cut (exactly one writer)
            ++rank;
        }
    }
}

__global__ void vox_offsets_kernel(const int* __restrict__ frame_m, int batch, int rows_cap,
                                   int* __restrict__ frame_rows, int* __restrict__ status) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        // every offset clamped to rows_cap: a frame that starts past the cap owns no rows, and frame_rows stays
        // non-decreasing and in range for the consumers that take per-frame row counts from it
        int acc = 0;
        for (int b = 0; b < batch; ++b) { frame_rows[b] = min(acc, rows_cap); acc += frame_m[b]; }
        if (acc > rows_cap) { atomicOr(status, SASSD_FLAG_VOXEL_CAP); acc = rows_cap; }
        frame_rows[batch] = acc;
    }
}

__global__ void __launch_bounds__(256)
vox_emit_kernel(const float4* __restrict__ points, const int* __restrict__ pt_off, int batch, VoxConst P,
                const int* __restrict__ pt_slot, const int* __restrict__ pt_next, const int* __restrict__ first,
                const int* __restrict__ head, const int* __restrict__ vid, const int* __restrict__ frame_cut,
                const int* __restrict__ frame_rows, int rows_cap, float4* __restrict__ voxels,
                int4* __restrict__ coors, int* __restrict__ num_points, float4* __restrict__ mean) {
    __shared__ int s_off[VOX_MAX_BATCH + 1];
    for (int b = threadIdx.x; b <= batch; b += blockDim.x) s_off[b] = pt_off[b];
    __syncthreads();
    const int n = s_off[batch];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int slot = __ldg(&pt_slot[i]);
        if (slot < 0 || __ldg(&first[slot]) != i) continue;
        const int b = sassd_frame_of(s_off, batch, i);
        const int cut = __ldg(&frame_cut[b]);
        if (i >= cut) continue;  // opener at/after the cut: its voxel id was never assigned
        const int v = __ldg(&vid[slot]);
        if (v < 0) continue;
        const int row = __ldg(&frame_rows[b]) + v;
        if (row >= rows_cap) continue;
        // the max_points smallest point indices below the cut, ascending
        int best[VOX_MAX_PTS];
        int cnt = 0;
        for (int j = __ldg(&head[slot]); j >= 0; j = __ldg(&pt_next[j])) {
            if (j >= cut) continue;
            int pos = cnt < P.max_points ? cnt : P.max_points;
            // insertion sort into best[0..min(cnt, max_points))
            if (pos == P.max_points) {
                if (j > best[P.max_points - 1]) { ++cnt; continue; }
                pos = P.max_points - 1;
            }
            while (pos > 0 && best[pos - 1] > j) { best[pos] = best[pos - 1]; --pos; }
            best[pos] = j;
            ++cnt;
        }
        const int num = cnt < P.max_points ? cnt : P.max_points;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s = 0; s < P.max_points; ++s) {
            float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
            if (s < num) q = __ldg(&points[best[s]]);
            voxels[(size_t)row * P.max_points + s] = q;
            acc.x += q.x; acc.y += q.y; acc.z += q.z; acc.w += q.w;
        }
        // cell of the opener (same arithmetic as the insert pass)
        const float4 p = __ldg(&points[i]);
        const int cx = (int)floorf(__fdiv_rn(__fsub_rn(p.x, P.lo[0]), P.vs[0]));
        const int cy = (int)floorf(__fdiv_rn(__fsub_rn(p.y, P.lo[1]), P.vs[1]));
        const int cz = (int)floorf(__fdiv_rn(__fsub_rn(p.z, P.lo[2]), P.vs[2]));
        coors[row] = make_int4(b, cz, cy, cx);
        num_points[row] = num;
        if (mean) {
            const float fn = (float)num;
            mean[row] = make_float4(__fdiv_rn(acc.x, fn), __fdiv_rn(acc.y, fn), __fdiv_rn(acc.z, fn),
                                    __fdiv_rn(acc.w, fn));
        }
    }
}

__global__ void voxel_mean_kernel(const float4* __restrict__ voxels, const int* __restrict__ num_points,
                                  const int* __restrict__ d_rows, int rows_cap, int max_points,
                                  float4* __restrict__ mean) {
    int rows = d_rows ? min(*d_rows, rows_cap) : rows_cap;
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s = 0; s < max_points; ++s) {
            float4 q = __ldg(&voxels[(size_t)r * max_points + s]);
            acc.x += q.x; acc.y += q.y; acc.z += q.z; acc.w += q.w;
        }
        const float fn = (float)num_points[r];
        mean[r] = make_float4(__fdiv_rn(acc.x, fn), __fdiv_rn(acc.y, fn), __fdiv_rn(acc.z, fn), __fdiv_rn(acc.w, fn));
    }
}

static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

extern "C" size_t sassd_voxelize_workspace_bytes(int n_points_cap, int batch, int slots_per_frame) {
    size_t t = (size_t)batch * slots_per_frame * sizeof(int);
    const size_t chunks_max = ((size_t)(n_points_cap > 0 ? n_points_cap : 1) + VR_CHUNK - 1) / VR_CHUNK;
    return 4 * align256(t) + 2 * align256((size_t)n_points_cap * sizeof(int)) + 2 * align256((size_t)batch * sizeof(int)) +
           align256((size_t)batch * chunks_max * sizeof(unsigned long long));
}

extern "C" int sassd_voxelize(const float* points, const int32_t* d_pt_off, int n_points_cap, int batch,
                              const sassd_voxel_params* hp, int slots_per_frame, float* voxels, int32_t* coors,
                              int32_t* num_points, float* mean, int rows_cap, int32_t* d_frame_rows,
                              int32_t* d_status, void* ws, size_t ws_bytes, sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!points || !d_pt_off || !hp || !voxels || !coors || !num_points || !d_frame_rows || !d_status || !ws)
        return SASSD_ERR_ARG;
    if (batch < 1 || batch > VOX_MAX_BATCH || hp->max_points < 1 || hp->max_points > VOX_MAX_PTS) return SASSD_ERR_ARG;
    if (slots_per_frame < 2 || (slots_per_frame & (slots_per_frame - 1))) return SASSD_ERR_ARG;
    if ((long long)hp->grid[0] * hp->grid[1] * hp->grid[2] >= 2147483647LL) return SASSD_ERR_UNSUPPORTED;
    if (ws_bytes < sassd_voxelize_workspace_bytes(n_points_cap, batch, slots_per_frame)) return SASSD_ERR_WORKSPACE;
    if (n_points_cap <= 0) n_points_cap = 1;

    size_t t = align256((size_t)batch * slots_per_frame * sizeof(int));
    size_t pn = align256((size_t)n_points_cap * sizeof(int));
    char* w = (char*)ws;
    int* keys = (int*)w; w += t;
    int* first = (int*)w; w += t;
    int* head = (int*)w; w += t;
    int* vid = (int*)w; w += t;
    int* pt_slot = (int*)w; w += pn;
    int* pt_next = (int*)w; w += pn;
    int* frame_m = (int*)w; w += align256((size_t)batch * sizeof(int));
    int* frame_cut = (int*)w; w += align256((size_t)batch * sizeof(int));
    unsigned long long* rank_desc = (unsigned long long*)w;
    const int chunks_max = (n_points_cap + VR_CHUNK - 1) / VR_CHUNK;

    VoxConst P;
    for (int j = 0; j < 3; ++j) { P.vs[j] = hp->voxel_size[j]; P.lo[j] = hp->range_min[j]; P.grid[j] = hp->grid[j]; }
    P.max_points = hp->max_points; P.max_voxels = hp->max_voxels;

    cudaMemsetAsync(keys, 0xff, t, stream);   // SASSD_EMPTY_KEY
    cudaMemsetAsync(first, 0x7f, t, stream);  // +inf
    cudaMemsetAsync(head, 0xff, t, stream);   // -1
    const int grid = sassd_grid(n_points_cap, 256);
    vox_insert_kernel<<<grid, 256, 0, stream>>>((const float4*)points, d_pt_off, batch, P, slots_per_frame, keys,
                                                first, head, pt_slot, pt_next, d_status, frame_m, frame_cut, rank_desc,
                                                batch * chunks_max);
    vox_rank_kernel<<<dim3(chunks_max, batch), 1024, 0, stream>>>(d_pt_off, pt_slot, first, vid, P.max_voxels, frame_m,
                                                                   frame_cut, rank_desc, chunks_max);
    vox_offsets_kernel<<<1, 32, 0, stream>>>(frame_m, batch, rows_cap, d_frame_rows, d_status);
    vox_emit_kernel<<<grid, 256, 0, stream>>>((const float4*)points, d_pt_off, batch, P, pt_slot, pt_next, first,
                                              head, vid, frame_cut, d_frame_rows, rows_cap, (float4*)voxels,
                                              (int4*)coors, num_points, (float4*)mean);
    return sassd_check_launch();
}

extern "C" int sassd_voxel_mean(const float* voxels, const int32_t* num_points, const int32_t* d_rows, int rows_cap,
                                int max_points, float* mean, sassd_stream_t stream_) {
    if (!voxels || !num_points || !mean || rows_cap < 0) return SASSD_ERR_ARG;
    if (rows_cap == 0) return SASSD_OK;
    voxel_mean_kernel<<<sassd_grid(rows_cap, 256), 256, 0, (cudaStream_t)stream_>>>(
        (const float4*)voxels, num_points, d_rows, rows_cap, max_points, (float4*)mean);
    return sassd_check_launch();
}

// ---------------------------------------------------------------------------
// anchors_mask: per-frame occupancy count map -> 2-D inclusive prefix sum ->
// 4-corner lookup per anchor.  int32 counts (the reference sums in fp32; counts
// <= 20000 are exact there, so the masks are identical).
// ---------------------------------------------------------------------------
__global__ void amask_count_kernel(const int4* __restrict__ coors, const int* __restrict__ d_rows, int rows_cap,
                                   int H, int W, int* __restrict__ map) {
    const int rows = min(*d_rows, rows_cap);
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
        const int4 c = __ldg(&coors[r]);  // (b, z, y, x)
        atomicAdd(&map[((size_t)c.x * H + c.z) * W + c.w], 1);
    }
}

// inclusive scan along x; one warp per row
__global__ void amask_rowscan_kernel(int* __restrict__ map, int nrows, int W) {
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < nrows; row += gridDim.x * wpb) {
        int* p = map + (size_t)row * W;
        int carry = 0;
        for (int x0 = 0; x0 < W; x0 += 32) {
            const int x = x0 + lane;
            int v = x < W ? p[x] : 0;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                int t = __shfl_up_sync(0xffffffffu, v, d);
                if (lane >= d) v += t;
            }
            v += carry;
            if (x < W) p[x] = v;
            carry = __shfl_sync(0xffffffffu, v, 31);
        }
    }
}

// inclusive scan along y; block = 32 columns x 32 row-groups, one strip of 32 columns per CTA
__global__ void __launch_bounds__(1024)
amask_colscan_kernel(int* __restrict__ map, int H, int W, int strips) {
    __shared__ int s_sum[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int b = blockIdx.x / strips, strip = blockIdx.x % strips;
    const int x = strip * 32 + tx;
    const int rpg = (H + 31) / 32;  // rows per group
    const int y0 = ty * rpg, y1 = min(y0 + rpg, H);
    int* p = map + (size_t)b * H * W;
    int acc = 0;
    if (x < W)
        for (int y = y0; y < y1; ++y) acc += p[(size_t)y * W + x];
    s_sum[ty][tx] = acc;
    __syncthreads();
    if (ty == 0) {
        int run = 0;
        for (int g = 0; g < 32; ++g) { int t = s_sum[g][tx]; s_sum[g][tx] = run; run += t; }
    }
    __syncthreads();
    if (x < W) {
        int run = s_sum[ty][tx];
        for (int y = y0; y < y1; ++y) { run += p[(size_t)y * W + x]; p[(size_t)y * W + x] = run; }
    }
}

__global__ void amask_lookup_kernel(const int* __restrict__ map, int H, int W, const int4* __restrict__ rects,
                                    int n_anchors, int batch, int threshold, uint8_t* __restrict__ mask) {
    const long long total = (long long)batch * n_anchors;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / n_anchors), a = (int)(i % n_anchors);
        const int4 r = __ldg(&rects[a]);  // c0 (x lo), c1 (y lo), c2 (x hi), c3 (y hi)
        const int* p = map + (size_t)b * H * W;
        // geometry.py:703-708: ID - IB - IC + IA on the inclusive integral image
        const int area = p[(size_t)r.w * W + r.z] - p[(size_t)r.w * W + r.x] - p[(size_t)r.y * W + r.z] +
                         p[(size_t)r.y * W + r.x];
        mask[i] = area > threshold ? 1 : 0;
    }
}

extern "C" size_t sassd_anchor_mask_workspace_bytes(int batch, int H, int W) {
    return (size_t)batch * H * W * sizeof(int);
}

extern "C" int sassd_anchor_mask(const int32_t* coors, const int32_t* d_rows, int rows_cap, int batch, int H, int W,
                                 const int32_t* rects, int n_anchors, int threshold, uint8_t* mask, void* ws,
                                 size_t ws_bytes, sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!coors || !d_rows || !rects || !mask || !ws || batch < 1) return SASSD_ERR_ARG;
    if (ws_bytes < sassd_anchor_mask_workspace_bytes(batch, H, W)) return SASSD_ERR_WORKSPACE;
    int* map = (int*)ws;
    cudaMemsetAsync(map, 0, (size_t)batch * H * W * sizeof(int), stream);
    amask_count_kernel<<<sassd_grid(rows_cap > 0 ? rows_cap : 1, 256), 256, 0, stream>>>((const int4*)coors, d_rows,
                                                                                          rows_cap, H, W, map);
    amask_rowscan_kernel<<<sassd_grid((long long)batch * H * 32, 256), 256, 0, stream>>>(map, batch * H, W);
    const int strips = (W + 31) / 32;
    amask_colscan_kernel<<<batch * strips, 1024, 0, stream>>>(map, H, W, strips);
    amask_lookup_kernel<<<sassd_grid((long long)batch * n_anchors, 256), 256, 0, stream>>>(
        map, H, W, (const int4*)rects, n_anchors, batch, threshold, mask);
    return sassd_check_launch();
}

extern "C" int sassd_version(void) { return 100; }

// launch hint of the tensor-core kernels (tc_common.cuh: launch_pdl)
namespace tc { int g_sassd_pdl = -1; }
extern "C" int sassd_set_pdl(int on) {
    const int prev = tc::g_sassd_pdl;
    tc::g_sassd_pdl = on;
    return prev;
}

// Rulebook construction for the spconv-v1 style sparse convolutions
// (SubMConv3d / SparseConv3d call sites: mmdet/models/necks/cmn.py:139-173,197-212).
//
// Hot-path representation: neighbour table nbr[n_out, 27] (output-stationary
// gather list).  The spconv-v1 pair tables are a re-indexing of it
// (sassd_rulebook_pairs) used at the API boundary and by the parity tests.
//
//  * hash index   : open addressing on the 31-bit flattened (b,z,y,x) key; one
//                   table per resolution level, shared by the SubM rulebook of
//                   that level and by the strided conv that consumes it.
//  * strided conv : every input marks the <= 8 output cells it feeds in a
//                   bitmap over the output grid (atomicOr); a popcount scan over
//                   the bitmap words yields the output rows already sorted by
//                   flattened index (the canonical order) — no sort, no
//                   thrust::unique, no dense int32 grid as in spconv v1.
//  * nbr fill     : one thread per (output row, offset) probes the input hash;
//                   a CTA stages one 128-row tile of the table in shared memory,
//                   writes it with one bulk (TMA) store and records which of the
//                   27 offsets occur in the tile (tile mask for tap skipping).
#include "common.cuh"

__device__ __forceinline__ int flat_key(int b, int z, int y, int x, int D, int H, int W) {
    return ((b * D + z) * H + y) * W + x;
}

__global__ void hash_build_kernel(const int4* __restrict__ coors, const int* __restrict__ d_rows, int rows_cap,
                                  int D, int H, int W, int* __restrict__ keys, int* __restrict__ vals, int slots,
                                  int* __restrict__ status) {
    const int rows = min(*d_rows, rows_cap);
    const uint32_t mask = (uint32_t)slots - 1u;
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
        const int4 c = __ldg(&coors[r]);
        const int key = flat_key(c.x, c.y, c.z, c.w, D, H, W);
        uint32_t s = sassd_hash32((uint32_t)key) & mask;
        int probes = 0;
        while (true) {
            int prev = atomicCAS(&keys[s], SASSD_EMPTY_KEY, key);
            if (prev == SASSD_EMPTY_KEY) { vals[s] = r; break; }
            if (prev == key) break;  // duplicate coordinate: first writer wins
            s = (s + 1) & mask;
            if (++probes >= slots) { atomicOr(status, SASSD_FLAG_HASH_FULL); break; }
        }
    }
}

extern "C" int sassd_hash_build(const int32_t* coors, const int32_t* d_rows, int rows_cap, int batch, int D, int H,
                                int W, int32_t* keys, int32_t* vals, int slots, int32_t* d_status,
                                sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!coors || !d_rows || !keys || !vals || !d_status) return SASSD_ERR_ARG;
    if (slots < 2 || (slots & (slots - 1)) || slots < 2 * rows_cap) return SASSD_ERR_ARG;
    if ((long long)batch * D * H * W >= 2147483647LL) return SASSD_ERR_UNSUPPORTED;
    cudaMemsetAsync(keys, 0xff, (size_t)slots * sizeof(int), stream);
    hash_build_kernel<<<sassd_grid(rows_cap > 0 ? rows_cap : 1, 256), 256, 0, stream>>>(
        (const int4*)coors, d_rows, rows_cap, D, H, W, keys, vals, slots, d_status);
    return sassd_check_launch();
}

// nbr[o*27 + k] = row of input cell  stride*o - pad + k  (stride=1,pad=1: SubM; stride=2,pad=1: strided).
// One CTA builds the table rows of one 128-row tile (SASSD_SPCONV_TILE_ROWS) in shared memory - one thread per
// (row, offset) probe of the input hash - and writes them with ONE bulk (TMA) store: the tile's rows are a contiguous
// 13.8 KB block of the table, so the write is fully coalesced and off the LSU.  While the entries are in flight the
// warps OR together which of the 27 offsets occur in the tile at all (ballot per offset is overkill: a warp-wide
// __reduce_or of the per-lane bit, then one shared atomicOr per warp); that 27-bit tile mask is what lets the sparse
// conv skip absent taps.
#define NBR_TILE_ROWS SASSD_SPCONV_TILE_ROWS
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src_smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src_smem), "r"(bytes) : "memory");
}
#define NBR_THREADS 1024      // 3456 probes per tile: <= 4 independent (latency-bound) hash probes in flight per thread
template <int STRIDE>
__global__ void __launch_bounds__(NBR_THREADS)
nbr_fill_kernel(const int4* __restrict__ coors_out, const int* __restrict__ d_rows, int rows_cap, int D, int H, int W,
                const int* __restrict__ keys, const int* __restrict__ vals, int slots, int* __restrict__ nbr,
                int* __restrict__ tile_mask) {
    __shared__ __align__(128) int s_tile[NBR_TILE_ROWS * 27];
    __shared__ unsigned int s_mask;
    const int rows = min(*d_rows, rows_cap);
    const int ntiles = (rows + NBR_TILE_ROWS - 1) / NBR_TILE_ROWS;
    const uint32_t mask = (uint32_t)slots - 1u;
    const uint32_t s_addr = (uint32_t)__cvta_generic_to_shared(s_tile);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        if (threadIdx.x == 0) s_mask = 0u;
        __syncthreads();
        const int row0 = tile * NBR_TILE_ROWS;
        const int rows_here = min(NBR_TILE_ROWS, rows_cap - row0);       // table rows this tile owns (capacity)
        unsigned int my_bits = 0u;
#pragma unroll 4
        for (int t = threadIdx.x; t < rows_here * 27; t += NBR_THREADS) {
            const int o = t / 27, k = t - o * 27;
            int res = -1;
            if (row0 + o < rows) {
                const int4 c = __ldg(&coors_out[row0 + o]);
                const int kz = k / 9, ky = (k / 3) % 3, kx = k % 3;
                const int z = c.y * STRIDE - 1 + kz, y = c.z * STRIDE - 1 + ky, x = c.w * STRIDE - 1 + kx;
                if (z >= 0 && z < D && y >= 0 && y < H && x >= 0 && x < W) {
                    const int slot = sassd_hash_find(keys, mask, flat_key(c.x, z, y, x, D, H, W));
                    if (slot >= 0) res = __ldg(&vals[slot]);
                }
            }
            s_tile[t] = res;
            if (res >= 0) my_bits |= 1u << k;
        }
        my_bits = __reduce_or_sync(0xffffffffu, my_bits);
        if ((threadIdx.x & 31) == 0 && my_bits) atomicOr(&s_mask, my_bits);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic writes -> visible to the bulk copy
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t bytes = (uint32_t)(rows_here * 27 * 4);
            const uint32_t bulk = bytes & ~15u;
            int* dst = nbr + (size_t)row0 * 27;
            if (bulk) bulk_s2g(dst, s_addr, bulk);
            for (uint32_t i = bulk / 4; i < bytes / 4; ++i) dst[i] = s_tile[i];       // < 16-byte tail of a ragged table
            if (tile_mask) tile_mask[tile] = (int)s_mask;
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");            // s_tile may be overwritten
        }
        __syncthreads();
    }
}

static int nbr_grid(int rows_cap) {
    const int tiles = sassd_div_up(rows_cap, NBR_TILE_ROWS);
    return tiles < sassd_num_sms() * 2 ? (tiles > 0 ? tiles : 1) : sassd_num_sms() * 2;
}

extern "C" int sassd_rulebook_subm(const int32_t* coors, const int32_t* d_rows, int rows_cap, int D, int H, int W,
                                   const int32_t* keys, const int32_t* vals, int slots, int32_t* nbr,
                                   int32_t* tile_mask, sassd_stream_t stream_) {
    if (!coors || !d_rows || !keys || !vals || !nbr) return SASSD_ERR_ARG;
    if (rows_cap <= 0) return SASSD_OK;
    nbr_fill_kernel<1><<<nbr_grid(rows_cap), NBR_THREADS, 0, (cudaStream_t)stream_>>>(
        (const int4*)coors, d_rows, rows_cap, D, H, W, keys, vals, slots, nbr, tile_mask);
    return sassd_check_launch();
}

extern "C" int sassd_rulebook_conv_nbr(const int32_t* coors_out, const int32_t* d_rows_out, int rows_cap_out, int D,
                                       int H, int W, const int32_t* keys_in, const int32_t* vals_in, int slots_in,
                                       int32_t* nbr, int32_t* tile_mask, sassd_stream_t stream_) {
    if (!coors_out || !d_rows_out || !keys_in || !vals_in || !nbr) return SASSD_ERR_ARG;
    if (rows_cap_out <= 0) return SASSD_OK;
    nbr_fill_kernel<2><<<nbr_grid(rows_cap_out), NBR_THREADS, 0, (cudaStream_t)stream_>>>(
        (const int4*)coors_out, d_rows_out, rows_cap_out, D, H, W, keys_in, vals_in, slots_in, nbr, tile_mask);
    return sassd_check_launch();
}

// ---------------------------------------------------------------------------
// strided conv output set (k=3, s=2, p=1)
// ---------------------------------------------------------------------------
#define BM_CHUNK 1024  // bitmap words per CTA of the compaction pass (one word per thread)

// Warp-aggregated marking: a warp covers 4 input rows x 8 candidate outputs; neighbouring inputs feed the same
// output cells, so lanes that hit the same bitmap word find each other (__match_any_sync), OR their bits in the warp
// and one lane issues the atomicOr.
__global__ void __launch_bounds__(256)
conv_mark_kernel(const int4* __restrict__ coors_in, const int* __restrict__ d_rows, int rows_cap,
                 int Do, int Ho, int Wo, uint32_t* __restrict__ bitmap) {
    const int rows = min(*d_rows, rows_cap);
    const long long total = (long long)rows * 8;
    const int lane = threadIdx.x & 31;
    for (long long t0 = blockIdx.x * (long long)blockDim.x + (threadIdx.x & ~31); t0 < total;
         t0 += (long long)gridDim.x * blockDim.x) {
        const long long t = t0 + lane;
        bool ok = t < total;
        int cell = 0;
        if (ok) {
            const int r = (int)(t >> 3), v = (int)(t & 7);
            const int4 c = __ldg(&coors_in[r]);
            // i = 2*o - 1 + k, k in {0,1,2}: odd i -> o in {(i+1)/2 (k=0), (i-1)/2 (k=2)}; even i -> o = i/2 (k=1)
            int oz, oy, ox;
            {
                const int i = c.y, sel = (v >> 2) & 1;
                if (i & 1) oz = sel ? (i - 1) >> 1 : (i + 1) >> 1; else { oz = i >> 1; ok &= (sel == 0); }
                ok &= (oz >= 0 && oz < Do);
            }
            {
                const int i = c.z, sel = (v >> 1) & 1;
                if (i & 1) oy = sel ? (i - 1) >> 1 : (i + 1) >> 1; else { oy = i >> 1; ok &= (sel == 0); }
                ok &= (oy >= 0 && oy < Ho);
            }
            {
                const int i = c.w, sel = v & 1;
                if (i & 1) ox = sel ? (i - 1) >> 1 : (i + 1) >> 1; else { ox = i >> 1; ok &= (sel == 0); }
                ok &= (ox >= 0 && ox < Wo);
            }
            if (ok) cell = flat_key(c.x, oz, oy, ox, Do, Ho, Wo);
        }
        const unsigned okmask = __ballot_sync(0xffffffffu, ok);
        if (ok) {
            const int word = cell >> 5;
            const unsigned peers = __match_any_sync(okmask, word);
            const uint32_t bits = __reduce_or_sync(peers, 1u << (cell & 31));
            if (lane == __ffs(peers) - 1) atomicOr(&bitmap[word], bits);
        }
    }
}

// Bitmap -> sorted output rows in ONE pass (round 1: count / scan / emit, three launches on the rulebook chain's
// critical path).  A CTA owns BM_CHUNK consecutive bitmap words, one per thread, so one block scan over the popcounts
// orders the rows by ascending cell index.  The chunk totals are chained by decoupled
// look-back: a CTA publishes {AGGREGATE, total}, walks back over its predecessors' descriptors until it meets an
// inclusive prefix and then publishes its own (CTAs are dispatched in index order, so the ones it waits for are
// running or done).  Each row is written and, when the caller passes the next level's hash table (keys pre-filled
// with SASSD_EMPTY_KEY), inserted into it on the spot - the separate sassd_hash_build launch of that level goes away.
// One bitmap word per thread: the thread that owns a solid run of cells emits at most 32 rows (with four words per
// thread a single thread wrote up to 128 rows one after the other while its CTA waited: 26 us per launch at B=1).
__global__ void __launch_bounds__(BM_CHUNK)
bm_compact_kernel(const uint32_t* __restrict__ bitmap, int nwords, unsigned long long* __restrict__ desc, int nchunks,
                  int Do, int Ho, int Wo, int rows_cap, int4* __restrict__ coors_out, int* __restrict__ d_rows_out,
                  int* __restrict__ keys, int* __restrict__ vals, int slots, int* __restrict__ status) {
    __shared__ int s_scan[33];
    __shared__ int s_base;
    const int c = blockIdx.x;
    const int w = c * BM_CHUNK + (int)threadIdx.x;
    uint32_t m = w < nwords ? __ldg(&bitmap[w]) : 0u;
    int total;
    const int ex = sassd_block_exscan(__popc(m), s_scan, &total);
    if (threadIdx.x < 32) {            // warp 0: publish, look back 32 predecessors at a time, publish the prefix
        volatile unsigned long long* vd = desc;
        const int lane = threadIdx.x;
        if (c > 0 && lane == 0) vd[c] = (SASSD_SCAN_AGG << 32) | (unsigned)total;
        const int base = sassd_lookback(vd, c, lane);
        if (lane == 0) {
            vd[c] = (SASSD_SCAN_PREFIX << 32) | (unsigned)(base + total);
            s_base = base;
            if (c == nchunks - 1) {
                int all = base + total;
                if (all > rows_cap) { atomicOr(status, SASSD_FLAG_ROWS_CAP); all = rows_cap; }
                *d_rows_out = all;
            }
        }
    }
    __syncthreads();
    const int base_row = s_base;
    if (m) {
        int row = base_row + ex;
        // (b, z, y, x) of the word's first cell; then walk with carries (no division per row)
        int cell0 = w * 32;
        int x = cell0 % Wo; cell0 /= Wo;
        int y = cell0 % Ho; cell0 /= Ho;
        int z = cell0 % Do;
        int b = cell0 / Do;
        int at = 0;                                              // cells advanced since (b, z, y, x) was computed
        while (m) {
            const int bit = __ffs(m) - 1;
            m &= m - 1;
            x += bit - at; at = bit;
            while (x >= Wo) { x -= Wo; if (++y == Ho) { y = 0; if (++z == Do) { z = 0; ++b; } } }
            if (row < rows_cap) coors_out[row] = make_int4(b, z, y, x);
            ++row;
        }
    }
    if (!keys) return;
    // Hash the chunk's rows with the whole CTA, one row per thread and round: an insertion is a chain of dependent L2
    // atomics, so a thread must not do the rows of its own word one after the other.
    __syncthreads();                                             // the rows above are visible to the CTA
    const uint32_t mask = (uint32_t)slots - 1u;
    const int nrows = min(total, max(rows_cap - base_row, 0));
    for (int i = threadIdx.x; i < nrows; i += blockDim.x) {
        const int row = base_row + i;
        const int4 cc = coors_out[row];
        const int key = flat_key(cc.x, cc.y, cc.z, cc.w, Do, Ho, Wo);      // unique: one row per marked cell
        uint32_t sl = sassd_hash32((uint32_t)key) & mask;
        int probes = 0;
        while (atomicCAS(&keys[sl], SASSD_EMPTY_KEY, key) != SASSD_EMPTY_KEY) {
            sl = (sl + 1) & mask;
            if (++probes >= slots) { atomicOr(status, SASSD_FLAG_HASH_FULL); break; }
        }
        if (probes < slots) vals[sl] = row;
    }
}

static inline size_t rb_align(size_t x) { return (x + 255) & ~(size_t)255; }

extern "C" size_t sassd_rulebook_conv_workspace_bytes(int batch, int Do, int Ho, int Wo) {
    const long long cells = (long long)batch * Do * Ho * Wo;
    const long long nwords = ((cells + 31) / 32 + 3) & ~3LL;
    const long long nchunks = (nwords + BM_CHUNK - 1) / BM_CHUNK;
    return rb_align((size_t)nwords * 4) + rb_align((size_t)nchunks * 8);
}

extern "C" int sassd_rulebook_conv_outputs_hash(const int32_t* coors_in, const int32_t* d_rows_in, int rows_cap_in,
                                                int batch, int D, int H, int W, int32_t* coors_out,
                                                int32_t* d_rows_out, int rows_cap_out, int32_t* keys_out,
                                                int32_t* vals_out, int slots_out, int32_t* d_status, void* ws,
                                                size_t ws_bytes, sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!coors_in || !d_rows_in || !coors_out || !d_rows_out || !d_status || !ws) return SASSD_ERR_ARG;
    if (keys_out && (!vals_out || slots_out < 2 || (slots_out & (slots_out - 1)) || slots_out < 2 * rows_cap_out))
        return SASSD_ERR_ARG;
    const int Do = (D + 2 - 3) / 2 + 1, Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const long long cells = (long long)batch * Do * Ho * Wo;
    if (cells >= 2147483647LL - 128) return SASSD_ERR_UNSUPPORTED;
    if (ws_bytes < sassd_rulebook_conv_workspace_bytes(batch, Do, Ho, Wo)) return SASSD_ERR_WORKSPACE;
    const int nwords = (int)(((cells + 31) / 32 + 3) & ~3LL);
    const int nchunks = (nwords + BM_CHUNK - 1) / BM_CHUNK;
    uint32_t* bitmap = (uint32_t*)ws;
    unsigned long long* desc = (unsigned long long*)((char*)ws + rb_align((size_t)nwords * 4));
    // one memset clears the bitmap and the chunk descriptors behind it
    cudaMemsetAsync(ws, 0, rb_align((size_t)nwords * 4) + (size_t)nchunks * 8, stream);
    if (keys_out) cudaMemsetAsync(keys_out, 0xff, (size_t)slots_out * sizeof(int), stream);
    conv_mark_kernel<<<sassd_grid((long long)(rows_cap_in > 0 ? rows_cap_in : 1) * 8, 256), 256, 0, stream>>>(
        (const int4*)coors_in, d_rows_in, rows_cap_in, Do, Ho, Wo, bitmap);
    bm_compact_kernel<<<nchunks, BM_CHUNK, 0, stream>>>(bitmap, nwords, desc, nchunks, Do, Ho, Wo, rows_cap_out,
                                                   (int4*)coors_out, d_rows_out, keys_out, vals_out, slots_out, d_status);
    return sassd_check_launch();
}

extern "C" int sassd_rulebook_conv_outputs(const int32_t* coors_in, const int32_t* d_rows_in, int rows_cap_in,
                                           int batch, int D, int H, int W, int32_t* coors_out, int32_t* d_rows_out,
                                           int rows_cap_out, int32_t* d_status, void* ws, size_t ws_bytes,
                                           sassd_stream_t stream_) {
    return sassd_rulebook_conv_outputs_hash(coors_in, d_rows_in, rows_cap_in, batch, D, H, W, coors_out, d_rows_out,
                                            rows_cap_out, nullptr, nullptr, 0, d_status, ws, ws_bytes, stream_);
}

// ---------------------------------------------------------------------------
// nbr -> spconv-v1 tables.  One CTA per kernel offset: ordered compaction over
// the output rows (canonical order: ascending output row).
// indice_pairs [2, 27, rows_cap] (-1 padded), indice_pair_num [27].
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
pairs_kernel(const int* __restrict__ nbr, const int* __restrict__ d_rows, int rows_cap, int* __restrict__ pairs,
             int* __restrict__ pair_num) {
    __shared__ int s_scan[33];
    const int k = blockIdx.x;
    const int rows = min(*d_rows, rows_cap);
    int* pin = pairs + (size_t)k * rows_cap;
    int* pout = pairs + (size_t)(27 + k) * rows_cap;
    int base = 0;
    for (int o0 = 0; o0 < rows; o0 += 1024) {
        const int o = o0 + threadIdx.x;
        const int i = o < rows ? nbr[(size_t)o * 27 + k] : -1;
        int total;
        const int pos = base + sassd_block_exscan(i >= 0 ? 1 : 0, s_scan, &total);
        if (i >= 0) { pin[pos] = i; pout[pos] = o; }
        base += total;
    }
    for (int p = base + threadIdx.x; p < rows_cap; p += 1024) { pin[p] = -1; pout[p] = -1; }
    if (threadIdx.x == 0) pair_num[k] = base;
}

extern "C" int sassd_rulebook_pairs(const int32_t* nbr, const int32_t* d_rows_out, int rows_cap,
                                    int32_t* indice_pairs, int32_t* indice_pair_num, sassd_stream_t stream_) {
    if (!nbr || !d_rows_out || !indice_pairs || !indice_pair_num || rows_cap <= 0) return SASSD_ERR_ARG;
    pairs_kernel<<<27, 1024, 0, (cudaStream_t)stream_>>>(nbr, d_rows_out, rows_cap, indice_pairs, indice_pair_num);
    return sassd_check_launch();
}

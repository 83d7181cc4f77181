// Ruled sparse convolution (SubMConv3d / SparseConv3d / 1x1x1; spconv v1.0 indice_conv semantics, call sites
// mmdet/models/necks/cmn.py:145-173,192-231) on the Hopper tensor cores (wgmma) with FP16x3 and the features kept in
// "split rows": two fp16 planes [2][rows_cap][C] (hi = half(x), lo = half((x - hi) * 2048)), C a multiple of 8.
//
// Structure (one CTA = one 128-row output tile at a time, output-stationary, no atomics, deterministic):
//   * 8 producer warps only *issue* 16-byte cp.async gathers (zero fill for missing neighbours) straight into the
//     128B-swizzled operand tiles plus an asynchronous mbarrier arrive; nobody waits for data.  Lane 0 of the first
//     producer warp also streams the weight blocks and the tile's [128,27] neighbour indices with cp.async.bulk.
//   * two consumer warpgroups (64 rows each) wait for the gathers, fence the generic->async proxy and issue
//     x*w = ah*bh + (ah*bl + al*bh)/2048 as wgmma (M = 64, N = BN, K = 16) into two register accumulators, then
//     run the epilogue (folded BN, ReLU, next layer's split planes and / or fp32 rows) from registers.
//   * narrow layers pack 2/4/8 taps into one 64-wide K chunk.
//   * tap skipping: the rulebook kernel records, per 128-row tile, which of the 27 taps have a neighbour
//     at all (tile_mask); chunks whose taps are all absent are skipped by every role - reference semantics only need
//     the listed pairs (spconv's indice_pairs), an absent pair contributes exactly zero.
//   * small layers (2 * tiles <= CTAs, i.e. one frame at a time): the two CTAs of a cluster split the active chunks
//     of ONE tile (split-K over taps); each hands the fp32 partial sums of the rows it does not finalise to its peer
//     through an L2-resident scratch row block and a remote mbarrier arrive (release/acquire at cluster scope).
#include "tc_common.cuh"

namespace sps {

using namespace tc;

constexpr int BKC = 64;                 // channels per chunk
constexpr int PROD_WARPS = 8;
constexpr int THREADS3 = CONS_THREADS + PROD_WARPS * 32;   // 512: 16 warps split evenly over the register file
constexpr int W_PROD = CONS_THREADS / 32;
constexpr int CLUSTER = 2;              // CTAs per cluster (tap split for small layers)
constexpr int SPLIT_TILES_MAX = 74;     // tiles of the scratch block (one per cluster: up to 148 CTAs per grid)

template <int BN>
struct Cfg3 {
    static constexpr int B_TILE_BYTES = BN * 128;
    static constexpr int STAGE_BYTES = 2 * A_TILE_BYTES + 2 * B_TILE_BYTES;
    static constexpr int STAGES = 4;
    static constexpr int NBR_TILE_BYTES = BM * 27 * 4;                    // one tile's rows of the [rows, 27] table
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * NBR_TILE_BYTES + 1024 + 512 + 256;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void st_shared_zero16(uint32_t dst) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(dst), "r"(0u) : "memory");
}
__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar) {   // arrive when this thread's prior cp.async land
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
// arrive (release, cluster scope) on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_remote(uint32_t bar, uint32_t rank) {
    asm volatile(
        "{\n\t"
        ".reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t"
        "}\n" ::"r"(bar), "r"(rank) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {    // acquire at cluster scope
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAITC_LOOP:\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra.uni WAITC_DONE;\n\t"
        "bra.uni WAITC_LOOP;\n\t"
        "WAITC_DONE:\n\t"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}

struct Args {
    const __half* in;       // [2][in_rows_cap][cin]
    size_t in_plane;        // elements between the hi and lo planes
    const void* wpack;
    const float* scale;
    const float* shift;
    const int* nbr;
    const int* tile_mask;   // [tiles] bit t = some row of the tile has a neighbour at tap t (null: all taps)
    const int* d_rows;
    __half* out_split;      // [2][rows_cap][out_ch] or null
    size_t out_plane;
    float* out_f32;         // [rows_cap][out_f32_stride] or null
    float* scratch;         // [SPLIT_TILES_MAX][128][BN] fp32 partial sums of the peer CTA (null: no tap split)
    int* counters;          // optional [2]: executed (tile, chunk) pairs, tiles (bench instrumentation)
    int cin, cout, taps, rows_cap, relu, out_ch, out_f32_stride;
};

// The chunks of one tile this CTA executes, identical in every role: chunk g is active when one of its taps is in the
// tile's mask; with a tap split the active chunks are dealt out alternately to the two CTAs of the cluster.
struct ChunkSet {
    uint32_t mask;     // bit g = chunk g is executed by this CTA
    __device__ __forceinline__ ChunkSet(uint32_t tap_mask, int tpg, int nchunks, int part, int nparts) {
        uint32_t act = tap_mask;
        if (tpg > 1) {
            const uint32_t group = (1u << tpg) - 1u;
            act = 0u;
            for (int g = 0; g < nchunks; ++g)
                if ((tap_mask >> (g * tpg)) & group) act |= 1u << g;
        }
        if (nparts == 1) { mask = act; return; }
        uint32_t m = 0u, rest = act;          // deal the active chunks out alternately (nparts == 2)
        for (int j = 0; rest; ++j) {
            const uint32_t low = rest & (0u - rest);
            if ((j & 1) == part) m |= low;
            rest ^= low;
        }
        mask = m;
    }
};

template <int TABLE, int BN>
__global__ void __cluster_dims__(CLUSTER, 1, 1) __launch_bounds__(THREADS3, 1) spconv_split_kernel(const Args p) {
    using C = Cfg3<BN>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
    const uint32_t nbr_base = base + C::STAGES * C::STAGE_BYTES;
    const int* nbr_smem = (const int*)(base_ptr + C::STAGES * C::STAGE_BYTES);
    const uint32_t bar_base = nbr_base + 2 * C::NBR_TILE_BYTES;
    auto full_a = [&](int s, int w) { return bar_base + 512u + 8u * (s * PROD_WARPS + w); };   // one per producer warp:
                                                                   // 32 async arrivals each, on separate words
    auto full_b = [&](int s) { return bar_base + 8u * (C::STAGES + s); };         // weight block landed
    auto empty = [&](int s) { return bar_base + 8u * (3 * C::STAGES + s); };
    auto nbr_full = [&](int b) { return bar_base + 8u * (4 * C::STAGES + 4 + b); };
    auto nbr_empty = [&](int b) { return bar_base + 8u * (4 * C::STAGES + 6 + b); };
    const uint32_t peer_done = bar_base + 8u * (4 * C::STAGES + 8);               // the peer's partial sums of my rows are in L2

    pdl_launch_dependents();      // the next layer may be scheduled as this grid's CTAs retire
    // warp index through a shuffle: the compiler then knows it is warp-uniform
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
    // Tap packing: a chunk is 64 K-columns = `tpg` taps of `cin` stored channels each (cin 8/16/32 -> 8/4/2 taps per
    // chunk), so the narrow early layers run 4/7/14 chunks per tile instead of 27.  The weight pack has the same
    // K order (sassd_spconv_pack).
    const int cin = p.cin;
    const int ppt = cin >> 3;                                // 16-byte pieces per tap
    const int tpg = (BKC % cin == 0) ? BKC / cin : 1;        // taps per chunk
    const int nchunks = (p.taps + tpg - 1) / tpg;
    const bool nbr_tiles = TABLE && p.taps <= 27;
    const uint32_t all_taps = p.taps >= 32 ? 0xffffffffu : ((1u << p.taps) - 1u);

    if (threadIdx.x == 0) {
        for (int s = 0; s < C::STAGES; ++s) {
            for (int w = 0; w < PROD_WARPS; ++w) mbar_init(full_a(s, w), 32);
            mbar_init(full_b(s), 1);
            mbar_init(empty(s), 2);                      // one arrive per consumer warpgroup
        }
        for (int b = 0; b < 2; ++b) { mbar_init(nbr_full(b), 1); mbar_init(nbr_empty(b), PROD_WARPS); }
        mbar_init(peer_done, 128);                       // the peer's giver warpgroup
        fence_barrier_init();
    }
    __syncthreads();
    cluster_sync_all();           // the peer's barriers exist before anyone arrives on them remotely
    pdl_wait();                   // producing layer / rulebook complete; nothing above touched global data
    const int M = p.d_rows ? min(__ldg(p.d_rows), p.rows_cap) : p.rows_cap;
    const int ntiles = (M + BM - 1) / BM;
    // Work decomposition, uniform over the grid: R full rounds of one tile per CTA, then the remaining `rem` tiles.  A
    // layer that has at most half as many tiles as there are CTAs (one frame at a time) runs as a TAP SPLIT: cluster q
    // owns tile q and its two CTAs share that tile's chunks, so a 45-tile layer occupies 90 SMs with half the chunk
    // chain each.  Splitting only the last partial round of a large layer does not pay: the hand-over at the very end
    // of the kernel overlaps nothing.  Hence R == 0.
    const uint32_t crank = cluster_ctarank();
    const int G = (int)gridDim.x;
    const int R = ntiles / G, rem = ntiles - R * G;
    const bool tail_split = TABLE && p.scratch && nchunks > 1 && R == 0 && rem > 0 && 2 * rem <= G &&
                            rem <= SPLIT_TILES_MAX;
    const int n_items = R + ((tail_split ? (int)(blockIdx.x >> 1) < rem : (int)blockIdx.x < rem) ? 1 : 0);
    struct Item { int tile, part, nparts; };
    auto item_at = [&](int i) {
        Item it;
        if (i < R) { it.tile = (int)blockIdx.x + i * G; it.part = 0; it.nparts = 1; }
        else if (tail_split) { it.tile = R * G + (int)(blockIdx.x >> 1); it.part = (int)crank; it.nparts = 2; }
        else { it.tile = R * G + (int)blockIdx.x; it.part = 0; it.nparts = 1; }
        return it;
    };
    auto chunks_of = [&](const Item& it) {
        uint32_t tm = all_taps;
        if (TABLE && p.tile_mask) {
            tm = (uint32_t)__ldg(&p.tile_mask[it.tile]) & all_taps;
            if (!tm) tm = 1u;       // a tile without any pair still has to produce act(shift): run one (all-zero) chunk
        }
        return ChunkSet(tm, tpg, nchunks, it.part, it.nparts).mask;
    };
    // Every CTA streams the same weight chunks.  If they all walked the taps in the same order they would ask the
    // same few L2 lines for the same 16 KB at the same time; each tile therefore starts at a different tap
    // (rotation by a tile-dependent offset, identical in all roles; the sum over taps is order-independent up to fp32
    // rounding and deterministic per tile).
    auto rot_of = [&](int tile) { return (int)(((unsigned)tile * 11u) % (unsigned)nchunks); };

    if (warp >= W_PROD) {
        // ===================== A producers: cp.async gather of split rows =====================
        // Nothing in this instruction stream waits for data: every thread issues its eight 16-byte copies (hardware
        // zero fill for a missing neighbour) and an asynchronous mbarrier arrive that fires when they have landed, so
        // the gather runs STAGES chunks ahead.  The 8 lanes of an octet copy the 8 pieces of ONE 128-byte row, so a
        // copy instruction touches 4 rows = 4 cache lines whatever the rows hold.
        const int pw = warp - W_PROD;                       // rows 16 pw .. 16 pw + 15
        const bool loader = pw == 0 && lane == 0;           // also streams weights and neighbour-table tiles
        const int piece = lane & 7, oct = lane >> 3;
        const int tl = piece / ppt, pc8 = (piece - tl * ppt) * 8;     // my tap within the chunk, element offset in it
        uint32_t offs[4];                                   // shared-memory offset of my 16 bytes of row j (any stage)
        int rowt[4];                                        // (row j) * taps
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = pw * 16 + j * 4 + oct;
            offs[j] = (uint32_t)(r >> 3) * 1024u + (uint32_t)(r & 7) * 128u + (((uint32_t)piece ^ (uint32_t)(r & 7)) << 4);
            rowt[j] = r * p.taps;
        }
        const __half* in_hi = p.in + pc8;
        const __half* in_lo = in_hi + p.in_plane;
        int stage = 0;
        uint32_t phase = 0;
        int nb = 0;                    // neighbour-table buffer of this tile
        uint32_t nb_phase = 0;
        int ld_nb = 0;                 // loader: next neighbour-table buffer to fill
        uint32_t ld_nb_phase = 0;
        auto load_nbr = [&](int tile) {     // one bulk copy: the tile's rows of the table are contiguous
            const int rows_here = min(BM, p.rows_cap - tile * BM);
            const uint32_t bytes = (uint32_t)(rows_here * p.taps * 4) & ~15u;
            mbar_wait(nbr_empty(ld_nb), ld_nb_phase ^ 1u);
            mbar_expect_tx(nbr_full(ld_nb), bytes);
            if (bytes) bulk_g2s(nbr_base + ld_nb * C::NBR_TILE_BYTES, p.nbr + (size_t)tile * BM * p.taps, bytes, nbr_full(ld_nb));
            if (++ld_nb == 2) { ld_nb = 0; ld_nb_phase ^= 1u; }
        };
        if (loader && nbr_tiles && n_items > 0) load_nbr(item_at(0).tile);
        for (int ii = 0; ii < n_items; ++ii) {
            const Item item = item_at(ii);
            const int tile = item.tile;
            // rows of the table the loader copied for this tile (whole 16-byte units only)
            const int rows_here = min(BM, p.rows_cap - tile * BM);
            const int rows_copied = nbr_tiles ? ((rows_here * p.taps * 4) & ~15) / (p.taps * 4) : 0;
            const int* ntile = nbr_smem + nb * (C::NBR_TILE_BYTES / 4);
            const uint32_t cmask = chunks_of(item);
            const int m0 = tile * BM + pw * 16 + oct;       // global row of j = 0
            if (nbr_tiles) {
                if (lane == 0) mbar_wait(nbr_full(nb), nb_phase);
                __syncwarp();
            }
            const int rot = rot_of(tile);
            auto chunk_at = [&](int gi) { return gi + rot < nchunks ? gi + rot : gi + rot - nchunks; };
            auto next_active = [&](int gi) {            // next position of the rotated walk whose chunk is executed
                for (++gi; gi < nchunks; ++gi)
                    if ((cmask >> chunk_at(gi)) & 1u) break;
                return gi;
            };
            // The neighbour indices are shared-memory loads through the same LSU queue as the cp.async copies, so
            // the indices of the NEXT chunk are requested BEFORE this chunk's copies are queued.
            auto load_srcs = [&](int g, int (&dst)[4]) {
                const int t = g * tpg + tl;
                const bool tap_ok = tl < tpg && t < p.taps;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int m = m0 + 4 * j;
                    dst[j] = -1;
                    if (tap_ok && m < M)
                        dst[j] = TABLE ? ((nbr_tiles && pw * 16 + j * 4 + oct < rows_copied) ? ntile[rowt[j] + t]
                                                                                          : __ldg(&p.nbr[(size_t)m * p.taps + t])) : m;
                }
            };
            int gi = next_active(-1);
            int srcs[4] = {-1, -1, -1, -1};
            if (gi < nchunks) load_srcs(chunk_at(gi), srcs);
            while (gi < nchunks) {
                const int gi_next = next_active(gi);
                // one lane polls the mbarrier, the warp follows
                if (lane == 0) {
                    mbar_wait(empty(stage), phase ^ 1u);
                    if (loader) {
                        const uint32_t dst = base + stage * C::STAGE_BYTES + 2 * A_TILE_BYTES;
                        const uint8_t* src = (const uint8_t*)p.wpack + (size_t)chunk_at(gi) * (2 * C::B_TILE_BYTES);
                        mbar_expect_tx(full_b(stage), 2 * C::B_TILE_BYTES);
                        bulk_g2s(dst, src, 2 * C::B_TILE_BYTES, full_b(stage));
                    }
                }
                __syncwarp();
                int nxt[4] = {-1, -1, -1, -1};
                if (gi_next < nchunks) load_srcs(chunk_at(gi_next), nxt);
                const uint32_t a_hi = base + stage * C::STAGE_BYTES, a_lo = a_hi + A_TILE_BYTES;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t nbytes = srcs[j] >= 0 ? 16u : 0u;     // 0 -> hardware zero fill
                    const uint32_t eo = (uint32_t)(srcs[j] < 0 ? 0 : srcs[j]) * (uint32_t)cin;
                    cp_async16(a_hi + offs[j], in_hi + eo, nbytes);
                    cp_async16(a_lo + offs[j], in_lo + eo, nbytes);
                }
                cp_async_arrive_noinc(full_a(stage, pw));
                if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
#pragma unroll
                for (int j = 0; j < 4; ++j) srcs[j] = nxt[j];
                gi = gi_next;
            }
            if (nbr_tiles) {
                __syncwarp();
                if (lane == 0) mbar_arrive(nbr_empty(nb));
                if (++nb == 2) { nb = 0; nb_phase ^= 1u; }
            }
            // The next tile's table goes into the buffer of tile ii - 1, which every producer warp has released long
            // before this warp has issued all of tile ii's copies: requested here, the wait costs nothing and warp 0
            // starts tile ii without waiting for the slowest warp of tile ii - 1.
            if (loader && nbr_tiles && ii + 1 < n_items) load_nbr(item_at(ii + 1).tile);
        }
    } else {
        // ===================== consumers: MMAs, then the epilogue from registers =====================
        const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
        float big[BN / 2], small[BN / 2];
        int stage = 0;
        uint32_t phase = 0;
        int executed = 0, tiles_done = 0;
        for (int ii = 0; ii < n_items; ++ii) {
            const Item item = item_at(ii);
            const int tile = item.tile, part = item.part;
            const bool split = item.nparts == 2;
            const uint32_t cmask = chunks_of(item);
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) { big[i] = 0.f; small[i] = 0.f; }
            const int rot = rot_of(tile);
            int prev = -1;
            for (int ci = 0; ci < nchunks; ++ci) {
                const int ch = ci + rot < nchunks ? ci + rot : ci + rot - nchunks;
                if (!((cmask >> ch) & 1u)) continue;
                // the gathers are generic-proxy writes (cp.async): fence before the MMAs read them
#pragma unroll 1
                for (int w = 0; w < PROD_WARPS; ++w) mbar_wait(full_a(stage, w), phase);
                fence_proxy_async();
                mbar_wait(full_b(stage), phase);
                const uint32_t ah = base + stage * C::STAGE_BYTES + (uint32_t)wg * (A_TILE_BYTES / 2);
                const uint32_t bh = base + stage * C::STAGE_BYTES + 2 * A_TILE_BYTES;
                wgmma_fence();
                // K columns past the chunk's last tap are zero in both operands (zero-filled gather, zero weight rows)
                mma_chunk_x3<1, BN>(big, small, ah, ah + A_TILE_BYTES, bh, bh + C::B_TILE_BYTES);
                wgmma_commit();
                wgmma_wait<1>();            // the previous chunk's MMAs have read their stage
                if (prev >= 0 && t == 0) mbar_arrive(empty(prev));
                prev = stage;
                ++executed;
                if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
            }
            wgmma_wait<0>();
            fence_regs<BN / 2>(big);
            fence_regs<BN / 2>(small);
            if (prev >= 0 && t == 0) mbar_arrive(empty(prev));
            if (part == 0) ++tiles_done;
            // Tap split: the two CTAs hold partial sums of the SAME 128 rows.  Each finalises half of them - CTA 0
            // rows 0..63 (warpgroup 0), CTA 1 rows 64..127 (warpgroup 1) - and its other warpgroup ("giver") hands
            // the partial sums of the rows it does not own to the peer: fp32 values in an L2-resident scratch block
            // at the positions of the (identical) register layout, then a remote mbarrier arrive (release / acquire
            // at cluster scope).  Half the bytes cross, in both directions at once, and the epilogue work is shared.
            const bool giver = split && wg != part;
            const int rl0 = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);    // tile rows rl0 and rl0 + 8
            float* prow = split ? p.scratch + (size_t)(tile - R * G) * BM * BN : nullptr;
            if (split && !giver) {              // keeper: the peer's partial sums of my rows must be visible
                mbar_wait_cluster(peer_done, 0u);
            }
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int n = 8 * j + 2 * (t & 3);
                const float scl0 = (p.scale && n < p.cout) ? __ldg(&p.scale[n]) : 1.f;
                const float scl1 = (p.scale && n + 1 < p.cout) ? __ldg(&p.scale[n + 1]) : 1.f;
                const float shl0 = (p.shift && n < p.cout) ? __ldg(&p.shift[n]) : 0.f;
                const float shl1 = (p.shift && n + 1 < p.cout) ? __ldg(&p.shift[n + 1]) : 0.f;
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int rl = rl0 + 8 * i, m = tile * BM + rl;
                    float a0 = __fadd_rn(big[4 * j + 2 * i], small[4 * j + 2 * i] * (1.f / kF16LoScale));
                    float a1 = __fadd_rn(big[4 * j + 2 * i + 1], small[4 * j + 2 * i + 1] * (1.f / kF16LoScale));
                    float2* q = split ? (float2*)(prow + (size_t)rl * BN + n) : nullptr;
                    if (giver) {                    // hand the partial sums over, no epilogue for these rows here
                        *q = make_float2(a0, a1);
                        continue;
                    }
                    if (split) {
                        const float2 pq = __ldcg(q);    // L2
                        a0 = __fadd_rn(a0, pq.x);
                        a1 = __fadd_rn(a1, pq.y);
                    }
                    // columns >= cout: zero weights, scale 1, shift 0 -> exactly 0
                    float o0 = fmaf(a0, scl0, shl0), o1 = fmaf(a1, scl1, shl1);
                    if (p.relu) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); }
                    if (m < M) {
                        if (p.out_f32 && n < p.out_f32_stride)
                            *(float2*)(p.out_f32 + (size_t)m * p.out_f32_stride + n) = make_float2(o0, o1);
                        if (p.out_split && 8 * j < p.out_ch) {
                            uint32_t h, l;
                            split_f16x2(o0, o1, h, l);
                            __half* ohi = p.out_split + (size_t)m * p.out_ch + n;
                            *(uint32_t*)ohi = h;
                            *(uint32_t*)(ohi + p.out_plane) = l;
                        }
                    }
                }
            }
            if (giver) mbar_arrive_remote(peer_done, (uint32_t)(part ^ 1));    // every thread releases its own stores
        }
        if (p.counters && threadIdx.x == 0 && executed) {
            atomicAdd(&p.counters[0], executed);
            atomicAdd(&p.counters[1], tiles_done);
        }
    }

    __syncthreads();
    cluster_sync_all();           // no CTA of the cluster exits while its peer may still arrive on its barriers
}

template <int TABLE, int BN>
static int launch3(const Args& a, cudaStream_t stream) {
    using C = Cfg3<BN>;
    auto kern = spconv_split_kernel<TABLE, BN>;
    // Persistent CTAs in clusters of two, one CTA per SM (~200 KB of shared memory): the grid must not exceed what is
    // co-resident - GPCs with an odd number of free SMs cannot host a last cluster, and a cluster left over for a
    // second wave would double the kernel's time.
    static int max_ctas = 0;
    if (!max_ctas) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES) != cudaSuccess)
            return SASSD_ERR_LAUNCH;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(CLUSTER * sassd_div_up(sassd_num_sms(), CLUSTER)); cfg.blockDim = dim3(THREADS3);
        cfg.dynamicSmemBytes = C::SMEM_BYTES;
        int clusters = 0;
        if (cudaOccupancyMaxActiveClusters(&clusters, kern, &cfg) != cudaSuccess || clusters < 1) {
            cudaGetLastError();
            clusters = sassd_num_sms() / (2 * CLUSTER);
        }
        max_ctas = CLUSTER * (clusters < SPLIT_TILES_MAX ? clusters : SPLIT_TILES_MAX);
    }
    // one CTA per tile up to the resident CTAs; with a tap split two CTAs per tile; always whole clusters
    int grid = CLUSTER * sassd_div_up(a.rows_cap, BM);
    if (grid > max_ctas) grid = max_ctas;
    if (launch_pdl(kern, dim3(grid), dim3(THREADS3), C::SMEM_BYTES, stream, a) != cudaSuccess) return SASSD_ERR_LAUNCH;
    return sassd_check_launch();
}

template <int TABLE>
static int dispatch3(const Args& a, cudaStream_t s) {
    if (a.cout <= 16) return launch3<TABLE, 16>(a, s);
    if (a.cout <= 32) return launch3<TABLE, 32>(a, s);
    if (a.cout <= 64) return launch3<TABLE, 64>(a, s);
    return SASSD_ERR_UNSUPPORTED;
}

}  // namespace sps

// Weight packer for sassd_spconv_f16x3: W [taps, cin, cout] fp32 -> per chunk [hi | lo][BN rows][64 K-columns] fp16,
// 128B-swizzled, K-column = (tap within chunk) * cin_stored + channel.
__global__ void spconv_pack_kernel(const float* __restrict__ w, int taps, int cin, int cs, int cout, int bn, int tpg,
                                   int nchunks, __half* __restrict__ out) {
    const long long per_chunk = 2LL * bn * 64;
    const long long total = (long long)nchunks * per_chunk;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int g = (int)(i / per_chunk);
        long long rem = i % per_chunk;
        const int part = (int)(rem / (bn * 64));          // 0 = hi, 1 = lo
        rem %= (bn * 64);
        const int n = (int)(rem / 64), pos = (int)(rem % 64);
        const int kk = (((pos >> 3) ^ (n & 7)) << 3) + (pos & 7);   // logical K-column stored at this physical slot
        const int tl = kk / cs, ch = kk % cs, t = g * tpg + tl;
        float v = 0.f;
        if (tl < tpg && t < taps && ch < cin && n < cout) v = w[((size_t)t * cin + ch) * cout + n];
        float hi, lo;
        tc::split_f16(v, hi, lo);
        out[i] = __float2half_rn(part == 0 ? hi : lo);
    }
}

static int spconv_bn(int cout) { return cout <= 16 ? 16 : (cout <= 32 ? 32 : 64); }
static int spconv_tpg(int cs) { return (64 % cs == 0) ? 64 / cs : 1; }

extern "C" size_t sassd_spconv_pack_bytes(int taps, int cin_stored, int cout) {
    if (taps < 1 || cin_stored < 8 || (cin_stored & 7) || cin_stored > 64 || cout < 1 || cout > 64) return 0;
    const int tpg = spconv_tpg(cin_stored);
    return (size_t)((taps + tpg - 1) / tpg) * 2 * spconv_bn(cout) * 128;
}

extern "C" int sassd_spconv_pack(const float* weight, int taps, int cin, int cin_stored, int cout, void* packed,
                                 sassd_stream_t stream_) {
    if (!weight || !packed || cin < 1 || cin > cin_stored || !sassd_spconv_pack_bytes(taps, cin_stored, cout))
        return SASSD_ERR_ARG;
    const int tpg = spconv_tpg(cin_stored), nchunks = (taps + tpg - 1) / tpg, bn = spconv_bn(cout);
    spconv_pack_kernel<<<sassd_grid((long long)nchunks * 2 * bn * 64, 256), 256, 0, (cudaStream_t)stream_>>>(
        weight, taps, cin, cin_stored, cout, bn, tpg, nchunks, (__half*)packed);
    return sassd_check_launch();
}

extern "C" size_t sassd_spconv_workspace_bytes(void) {
    // fp32 partial sums of the peer CTA for the tap split: SPLIT_TILES_MAX tiles x 128 rows x 64 columns
    return (size_t)sps::SPLIT_TILES_MAX * sps::BM * 64 * sizeof(float);
}

extern "C" int sassd_spconv_f16x3(const sassd_spconv_desc* d, const void* in_split, const void* wpack,
                                  const float* scale, const float* shift, const int32_t* nbr,
                                  const int32_t* tile_mask, const int32_t* d_rows, void* out_split, float* out_f32,
                                  void* ws, size_t ws_bytes, int32_t* counters, sassd_stream_t stream_) {
    if (!d || !in_split || !wpack || (!out_split && !out_f32)) return SASSD_ERR_ARG;
    if (d->cin < 8 || (d->cin & 7) || d->cin > 64 || d->cout < 1 || d->cout > 64 || d->taps < 1 || d->rows_cap < 0)
        return SASSD_ERR_ARG;
    if (d->taps > 1 && !nbr) return SASSD_ERR_ARG;
    if (tile_mask && d->taps > 27) return SASSD_ERR_ARG;
    if (out_split && ((d->out_ch & 7) || d->out_ch < d->cout)) return SASSD_ERR_ARG;
    if (out_f32 && (d->out_f32_stride & 3)) return SASSD_ERR_ARG;
    if (ws && ws_bytes < sassd_spconv_workspace_bytes()) return SASSD_ERR_WORKSPACE;
    if (d->rows_cap == 0) return SASSD_OK;
    sps::Args a;
    a.in = (const __half*)in_split; a.in_plane = (size_t)d->in_rows_cap * d->cin;
    a.wpack = wpack; a.scale = scale; a.shift = shift; a.nbr = nbr; a.tile_mask = tile_mask; a.d_rows = d_rows;
    a.out_split = (__half*)out_split; a.out_plane = (size_t)d->rows_cap * d->out_ch; a.out_f32 = out_f32;
    a.scratch = (float*)ws; a.counters = counters;
    a.cin = d->cin; a.cout = d->cout; a.taps = d->taps; a.rows_cap = d->rows_cap; a.relu = d->relu;
    a.out_ch = d->out_ch; a.out_f32_stride = d->out_f32_stride;
    return d->taps > 1 ? sps::dispatch3<1>(a, (cudaStream_t)stream_) : sps::dispatch3<0>(a, (cudaStream_t)stream_);
}

// fp32 rows [rows, cin] -> split rows [2][rows_cap][cs] (cs >= cin, multiple of 8; padding channels zero)
__global__ void features_to_split_kernel(const float* __restrict__ feat, const int* __restrict__ d_rows, int rows_cap,
                                         int cin, int cs, __half* __restrict__ out) {
    const int rows = d_rows ? min(*d_rows, rows_cap) : rows_cap;
    const long long total = (long long)rows * cs;
    const size_t plane = (size_t)rows_cap * cs;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i / cs), c = (int)(i % cs);
        float hi = 0.f, lo = 0.f;
        if (c < cin) tc::split_f16(feat[(size_t)r * cin + c], hi, lo);
        out[i] = __float2half_rn(hi);
        out[i + plane] = __float2half_rn(lo);
    }
}

extern "C" int sassd_features_to_split(const float* feat, const int32_t* d_rows, int rows_cap, int cin, int cs,
                                       void* out_split, sassd_stream_t stream_) {
    if (!feat || !out_split || cin < 1 || cs < cin || (cs & 7)) return SASSD_ERR_ARG;
    if (rows_cap <= 0) return SASSD_OK;
    features_to_split_kernel<<<sassd_grid((long long)rows_cap * cs, 256), 256, 0, (cudaStream_t)stream_>>>(
        feat, d_rows, rows_cap, cin, cs, (__half*)out_split);
    return sassd_check_launch();
}

// dense(): split rows [2][rows_cap][C] -> split BEV map [2][B][H][W][D*C] (channel d*C + c), 16 bytes per thread
__global__ void split_rows_to_bev_kernel(const uint4* __restrict__ feat, size_t in_plane16, const int4* __restrict__ coors,
                                         const int* __restrict__ d_rows, int rows_cap, int C8, int D, int H, int W,
                                         size_t out_plane16, uint4* __restrict__ bev, int* __restrict__ tile_dist) {
    const int rows = min(*d_rows, rows_cap);
    const long long total = (long long)rows * C8;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i / C8), q = (int)(i % C8);
        const int4 c = __ldg(&coors[r]);
        const size_t o = (((size_t)c.x * H + c.z) * W + c.w) * (size_t)(D * C8) + (size_t)c.y * C8 + q;
        bev[o] = __ldg(&feat[i]);
        bev[o + out_plane16] = __ldg(&feat[i + in_plane16]);
        if (tile_dist && q == 0) sassd_mark_conv2d_tiles(tile_dist, c.x, c.z, c.w, H, W);
    }
}

extern "C" int sassd_split_rows_to_bev(const void* feat_split, const int32_t* coors, const int32_t* d_rows, int rows_cap,
                                       int C, int D, int H, int W, int batch, void* bev_split, int32_t* tile_dist,
                                       sassd_stream_t stream_) {
    if (!feat_split || !coors || !d_rows || !bev_split || (C & 7) || batch < 1) return SASSD_ERR_ARG;
    if (rows_cap <= 0) return SASSD_OK;
    const size_t in_plane16 = (size_t)rows_cap * C / 8, out_plane16 = (size_t)batch * H * W * D * C / 8;
    split_rows_to_bev_kernel<<<sassd_grid((long long)rows_cap * (C / 8), 256), 256, 0, (cudaStream_t)stream_>>>(
        (const uint4*)feat_split, in_plane16, (const int4*)coors, d_rows, rows_cap, C / 8, D, H, W, out_plane16,
        (uint4*)bev_split, tile_dist);
    return sassd_check_launch();
}

// Dense NHWC 3x3 / 1x1 convolution + folded BatchNorm + ReLU for the BEV neck and the heads
// (BEVNet cmn.py:233-282, SSDRotateHead ssd_rotate_head.py:218-231, PSWarpHead.convs :424-429),
// Hopper tensor cores (wgmma) on FP16x3, with the activation operand moved by TMA.
//
// Why a second tensor-core kernel: in gconv_tc.cu the A operand is gathered by producer warps
// (LDG -> split -> STS), nine times per element for a 3x3 conv.  Here
//   * activations live in HBM already split: two fp16 planes [2][B][H][W][C] (hi, lo*2048), written
//     once by the epilogue of the producing layer (or by the sparse->BEV scatter);
//   * a tile is an 8x16-pixel patch; for tap (dy,dx) and a 64-channel chunk the A operand is ONE
//     cp.async.bulk.tensor.4d box {64 ch, 16 x, 8 y, 1} at (y0+dy, x0+dx) — TMA writes it 128B-swizzled
//     straight into the wgmma operand layout and zero-fills out-of-image pixels (= the conv's zero padding);
//   * no producer warps: warp 8 lane 0 issues the TMA boxes (A hi, A lo) and the weight bulk copies, two consumer
//     warpgroups (pixel rows 0-63 / 64-127 of the tile) issue the MMAs and store the outputs from registers.
// A work unit is a tile and up to 128 of its output channels: the two register accumulators (big, small) of a
// 64 x 128 block are 128 floats per thread, so 256-channel layers run each tile as two units on the same weight pack.
#include <cuda.h>

#include <cstdlib>

#include "tc_common.cuh"

namespace tma {

using namespace tc;

constexpr int TILE_H = SASSD_CONV2D_TILE_H, TILE_W = SASSD_CONV2D_TILE_W;   // 8 x 16 = 128 output pixels per tile
constexpr int BKC = 64;                         // channels per chunk (one 128-byte fp16 row)
constexpr int kConstTile = 1 << 30;             // tile reference flag: the tile only stores the layer's constant vector
constexpr int CONS_WARPS = CONS_THREADS / 32;   // 8
constexpr int THREADS2 = CONS_THREADS + 32;     // + the TMA / bulk-copy issuing warp
constexpr int W_LOAD = CONS_WARPS;

template <int BN>
struct Cfg2 {
    static constexpr int B_TILE_BYTES = BN * 128;
    static constexpr int STAGE_BYTES = 2 * A_TILE_BYTES + 2 * B_TILE_BYTES;
    static constexpr int STAGES = (BN >= 128) ? 3 : (BN >= 64 ? 4 : 5);
    // tile order (active tiles first) when the map carries constant-region information: uint16 per tile
    static constexpr int ORDER_CAP = 832;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256 + ORDER_CAP * 2;
};

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
        ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar)
        : "memory");
}

struct Conv2dArgs {
    const void* wpack;
    const float* scale;
    const float* shift;
    float* out_f32;       // [B,H,W,out_f32_stride] or null
    __half* out_split;    // [2,B,H,W,out_split_ch] or null
    int batch, H, W, cin, cout, taps, relu, out_f32_stride, out_split_ch;
    const int* tile_dist; // optional: distance of each tile to the nearest active cell of the scattered map
    const float* cvec;    // output constant of the tiles that see a constant input (tile_dist > reach, not on the border)
    int reach;
    int* counters;        // optional [2]: += tiles computed (not stored as a constant), += tiles (bench instrumentation)
    int tile_order;       // 1: computed tiles first, 0: round-robin
    int nsplit;           // work units per tile: 1, or 2 = each unit computes BN of the 2*BN output channels (the weight
                          // pack is the 2*BN-wide one)
};

// True when tile (ty, tx) sees a constant input and its output is p.cvec (see sassd_conv2d_f16x3_occ in the header).
__device__ __forceinline__ bool tile_is_constant(const Conv2dArgs& p, int tile, int ty, int tx, int tiles_y, int tiles_x) {
    if (!p.tile_dist || __ldg(&p.tile_dist[tile]) <= p.reach) return false;
    return p.reach < 2 || !(ty == 0 || ty == tiles_y - 1 || tx == 0 || tx == tiles_x - 1);
}

// A unit of a constant-region tile: every pixel gets the layer's constant vector (channels [n_off, n_off + ncols) of it).
// Lane g of a pixel's group holds 8 channels of the split constant in registers and the EW consumer warps write
// whole pixels with 16-byte stores (ncols / 8 lanes cover one pixel: 512 contiguous bytes at ncols = 256).  Same
// values, bit for bit, as the register epilogue of a constant tile.  Requires vpp = ncols / 8 in {8, 16, 32}.
template <int EW>
__device__ __forceinline__ void store_constant_unit(const Conv2dArgs& p, int b, int ty, int tx, int n_off, int ncols,
                                                    int warp, int lane) {
    const int vpp = ncols >> 3, g = lane % vpp, sub = lane / vpp, ppi = 32 / vpp;
    const int c = n_off + 8 * g;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (c + j) < p.cout ? __ldg(&p.cvec[c + j]) : 0.f;
    uint4 hi, lo;
    split_f16x2(v[0], v[1], hi.x, lo.x);
    split_f16x2(v[2], v[3], hi.y, lo.y);
    split_f16x2(v[4], v[5], hi.z, lo.z);
    split_f16x2(v[6], v[7], hi.w, lo.w);
    const size_t plane = (size_t)p.batch * p.H * p.W * p.out_split_ch;
#pragma unroll 4
    for (int pg = warp; pg * ppi < TILE_H * TILE_W; pg += EW) {
        const int pix = pg * ppi + sub;
        const int y = ty * TILE_H + pix / TILE_W, x = tx * TILE_W + pix % TILE_W;
        if (y < p.H && x < p.W) {
            __half* dst = p.out_split + (((size_t)b * p.H + y) * p.W + x) * p.out_split_ch + c;
            *(uint4*)dst = hi;
            *(uint4*)(dst + plane) = lo;
        }
    }
}

template <int BN>
__global__ void __launch_bounds__(THREADS2, 1)
conv2d_tma_kernel(const __grid_constant__ CUtensorMap amap, const Conv2dArgs p) {
    using C = Cfg2<BN>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
    const uint32_t bar_base = base + C::STAGES * C::STAGE_BYTES;
    auto full = [&](int s) { return bar_base + 8u * s; };
    auto empty = [&](int s) { return bar_base + 8u * (C::STAGES + s); };

    pdl_launch_dependents();      // the next layer may be scheduled as this grid's CTAs retire
    // warp index through a shuffle so that the compiler knows it is warp-uniform
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
    const int tiles_x = (p.W + TILE_W - 1) / TILE_W, tiles_y = (p.H + TILE_H - 1) / TILE_H;
    const int ntiles = p.batch * tiles_y * tiles_x;
    const int nsplit = p.nsplit, nunits = ntiles * nsplit;      // work unit k: tile k / nsplit, output channels (k % nsplit) * BN ...
    const int kchunks = (p.cin + BKC - 1) / BKC;
    const int nchunks = p.taps * kchunks;

    if (threadIdx.x == 0) {
        for (int s = 0; s < C::STAGES; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), 2); }
        fence_barrier_init();
        asm volatile("prefetch.tensormap [%0];" ::"l"(&amap) : "memory");
    }
    __syncthreads();
    pdl_wait();                   // the producing layer has completed; nothing above touched global data

    // With constant-region information most tiles only store a constant.  Static round-robin leaves some CTAs with
    // two computed tiles and others with none; with tile_order = 1 (for maps of up to ORDER_CAP tiles) every CTA
    // builds the same order - computed tiles first, constant tiles after - and all roles walk
    // order[blockIdx.x + i * gridDim.x].  Round-robin is the default: with several steps in flight the SMs that
    // only store constants are what the other frames' kernels run on.
    uint16_t* order = (uint16_t*)(base_ptr + C::STAGES * C::STAGE_BYTES + 256);
    const bool small_map = p.tile_dist != nullptr && ntiles <= C::ORDER_CAP;
    const bool use_order = p.tile_order && small_map;
    // For maps of up to ORDER_CAP tiles warp 0 fetches every tile's distance in one batch of loads (one memory latency
    // instead of one per tile and role) and keeps the verdicts as order[k] bit 15.
    if (small_map) {
        if (warp == 0) {
            // verdicts of tiles lane, lane + 32, ... as bits of one word; the distances are fetched four at a time
            uint32_t cst_bits = 0u;
            int ty = (lane / tiles_x) % tiles_y, tx = lane % tiles_x;      // tile `lane`; advanced by 32 tiles per slot
#pragma unroll 1
            for (int i0 = 0; i0 * 32 < ntiles; i0 += 4) {
                int dist[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int t = (i0 + e) * 32 + lane;
                    dist[e] = t < ntiles ? __ldg(&p.tile_dist[t]) : 0;
                }
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int t = (i0 + e) * 32 + lane;
                    const bool border = ty == 0 || ty == tiles_y - 1 || tx == 0 || tx == tiles_x - 1;   // sees the zero padding
                    if (t < ntiles && dist[e] > p.reach && (p.reach < 2 || !border)) cst_bits |= 1u << (i0 + e);
                    tx += 32;
                    while (tx >= tiles_x) { tx -= tiles_x; if (++ty == tiles_y) ty = 0; }
                }
            }
            if (use_order) {
                int n = 0;
                for (int pass = 0; pass < 2; ++pass)
#pragma unroll 1
                    for (int i = 0; i * 32 < ntiles; ++i) {
                        const int t = i * 32 + lane;
                        const bool cst = (cst_bits >> i) & 1u;
                        const bool take = t < ntiles && (cst == (pass == 1));
                        const uint32_t m = __ballot_sync(0xffffffffu, take);
                        if (take) order[n + __popc(m & ((1u << lane) - 1u))] = (uint16_t)(t | (cst ? 0x8000 : 0));
                        n += __popc(m);
                    }
            } else {
#pragma unroll 1
                for (int i = 0; i * 32 < ntiles; ++i) {
                    const int t = i * 32 + lane;
                    if (t < ntiles) order[t] = (uint16_t)(t | (((cst_bits >> i) & 1u) ? 0x8000 : 0));
                }
            }
        }
        __syncthreads();
    }
    // tile_ref(k): the k-th tile in walking order, bit 30 set when it only stores the layer's constant
    auto tile_ref = [&](int k) -> int {
        if (small_map) { const int v = order[k]; return (v & 0x7fff) | ((v & 0x8000) << 15); }
        if (!p.tile_dist) return k;
        return tile_is_constant(p, k, (k / tiles_x) % tiles_y, k % tiles_x, tiles_y, tiles_x) ? (k | kConstTile) : k;
    };

    if (warp == W_LOAD) {
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int k = blockIdx.x; k < nunits; k += gridDim.x) {
                const int ref = tile_ref(k / nsplit), half = k % nsplit;
                if (ref & kConstTile) continue;                                         // nothing to load
                const int tile = ref;
                const int b = tile / (tiles_y * tiles_x);
                const int ty = (tile / tiles_x) % tiles_y, tx = tile % tiles_x;
                const int y0 = ty * TILE_H, x0 = tx * TILE_W;
                for (int t = 0; t < p.taps; ++t) {
                    const int dy = p.taps == 9 ? t / 3 - 1 : 0, dx = p.taps == 9 ? t % 3 - 1 : 0;
                    for (int kc = 0; kc < kchunks; ++kc) {
                        mbar_wait(empty(stage), phase ^ 1u);
                        const uint32_t a_hi = base + stage * C::STAGE_BYTES, a_lo = a_hi + A_TILE_BYTES;
                        const uint32_t b_dst = a_hi + 2 * A_TILE_BYTES;
                        mbar_expect_tx(full(stage), 2 * A_TILE_BYTES + 2 * C::B_TILE_BYTES);
                        // coordinates innermost first: {channel, x, y, plane*B + b}; out-of-image pixels arrive as zeros
                        tma_load_4d(a_hi, &amap, kc * BKC, x0 + dx, y0 + dy, b, full(stage));
                        tma_load_4d(a_lo, &amap, kc * BKC, x0 + dx, y0 + dy, p.batch + b, full(stage));
                        // pack: per (tap, chunk) [hi | lo], each nsplit * BN rows of 128 bytes; this unit's BN rows of each
                        const uint8_t* src = (const uint8_t*)p.wpack +
                                             (size_t)(t * kchunks + kc) * (size_t)(2 * nsplit) * C::B_TILE_BYTES +
                                             (size_t)half * C::B_TILE_BYTES;
                        constexpr uint32_t kPiece = (C::B_TILE_BYTES >= 8192) ? 8192u : (uint32_t)C::B_TILE_BYTES;
#pragma unroll 1
                        for (int part = 0; part < 2; ++part)
#pragma unroll 1
                            for (uint32_t o = 0; o < (uint32_t)C::B_TILE_BYTES; o += kPiece)
                                bulk_g2s(b_dst + part * C::B_TILE_BYTES + o,
                                         src + (size_t)part * nsplit * C::B_TILE_BYTES + o, kPiece, full(stage));
                        if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
                    }
                }
            }
        }
    } else {
        // ===================== consumers: warpgroup wg owns pixel rows 64 wg .. 64 wg + 63 of the tile =====================
        const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
        const int rl0 = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);        // tile rows rl0 and rl0 + 8 (= pixel py * 16 + px)
        const size_t plane = (size_t)p.batch * p.H * p.W * p.out_split_ch;
        float big[BN / 2], small[BN / 2];
        int stage = 0;
        uint32_t phase = 0;
        int computed = 0;
        for (int k = blockIdx.x; k < nunits; k += gridDim.x) {
            const int ref = tile_ref(k / nsplit), n_off = (k % nsplit) * BN;
            const int tile = ref & ~kConstTile;
            const bool const_tile = (ref & kConstTile) != 0;
            const int b = tile / (tiles_y * tiles_x);
            const int ty = (tile / tiles_x) % tiles_y, tx = tile % tiles_x;
            if (const_tile) {                                               // no MMAs run for this tile
                const int ncols = min(BN, p.out_split_ch - n_off);
                if (p.out_split && !p.out_f32 && (ncols == 64 || ncols == 128 || ncols == 256)) {
                    store_constant_unit<CONS_WARPS>(p, b, ty, tx, n_off, ncols, warp, lane);
                    continue;
                }
            } else {
                if (k % nsplit == 0) ++computed;
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) { big[i] = 0.f; small[i] = 0.f; }
                int prev = -1;
                for (int ch = 0; ch < nchunks; ++ch) {
                    mbar_wait(full(stage), phase);
                    const uint32_t ah = base + stage * C::STAGE_BYTES + (uint32_t)wg * (A_TILE_BYTES / 2);
                    const uint32_t bh = base + stage * C::STAGE_BYTES + 2 * A_TILE_BYTES;
                    wgmma_fence();
                    mma_chunk_x3<1, BN>(big, small, ah, ah + A_TILE_BYTES, bh, bh + C::B_TILE_BYTES);
                    wgmma_commit();
                    wgmma_wait<1>();            // the previous chunk's MMAs have read their stage
                    if (prev >= 0 && t == 0) mbar_arrive(empty(prev));
                    prev = stage;
                    if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
                }
                wgmma_wait<0>();
                fence_regs<BN / 2>(big);
                fence_regs<BN / 2>(small);
                if (prev >= 0 && t == 0) mbar_arrive(empty(prev));
            }
            // epilogue from registers: folded BN + ReLU (or the layer constant), fp32 and / or split-plane stores
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int n = n_off + 8 * j + 2 * (t & 3);
                float c0, c1, sc0 = 1.f, sc1 = 1.f, sh0 = 0.f, sh1 = 0.f;
                if (const_tile) {
                    c0 = n < p.cout ? __ldg(&p.cvec[n]) : 0.f;
                    c1 = n + 1 < p.cout ? __ldg(&p.cvec[n + 1]) : 0.f;
                } else {
                    if (p.scale && n < p.cout) sc0 = __ldg(&p.scale[n]);
                    if (p.scale && n + 1 < p.cout) sc1 = __ldg(&p.scale[n + 1]);
                    if (p.shift && n < p.cout) sh0 = __ldg(&p.shift[n]);
                    if (p.shift && n + 1 < p.cout) sh1 = __ldg(&p.shift[n + 1]);
                }
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int rl = rl0 + 8 * i;
                    const int y = ty * TILE_H + rl / TILE_W, x = tx * TILE_W + rl % TILE_W;
                    float o0 = c0, o1 = c1;
                    if (!const_tile) {
                        o0 = fmaf(__fadd_rn(big[4 * j + 2 * i], small[4 * j + 2 * i] * (1.f / kF16LoScale)), sc0, sh0);
                        o1 = fmaf(__fadd_rn(big[4 * j + 2 * i + 1], small[4 * j + 2 * i + 1] * (1.f / kF16LoScale)), sc1, sh1);
                        if (p.relu) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); }
                        if (n >= p.cout) o0 = 0.f;
                        if (n + 1 >= p.cout) o1 = 0.f;
                    }
                    if (y >= p.H || x >= p.W) continue;
                    const size_t pix = ((size_t)b * p.H + y) * p.W + x;
                    if (p.out_f32 && n < p.out_f32_stride)
                        *(float2*)(p.out_f32 + pix * p.out_f32_stride + n) = make_float2(o0, o1);
                    if (p.out_split && n < p.out_split_ch) {
                        uint32_t h, l;
                        split_f16x2(o0, o1, h, l);
                        __half* dst = p.out_split + pix * p.out_split_ch + n;
                        *(uint32_t*)dst = h;
                        *(uint32_t*)(dst + plane) = l;
                    }
                }
            }
        }
        if (p.counters && threadIdx.x == 0) {
            if (computed) atomicAdd(&p.counters[0], computed);
            if (blockIdx.x == 0) atomicAdd(&p.counters[1], ntiles);
        }
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

template <int BN>
static int launch2(const CUtensorMap& map, const Conv2dArgs& a, cudaStream_t stream) {
    using C = Cfg2<BN>;
    auto kern = conv2d_tma_kernel<BN>;
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES) != cudaSuccess)
            return SASSD_ERR_LAUNCH;
        configured = true;
    }
    const int units = a.batch * sassd_div_up(a.H, TILE_H) * sassd_div_up(a.W, TILE_W) * a.nsplit;
    const int grid = units < sassd_num_sms() ? units : sassd_num_sms();
    if (launch_pdl(kern, dim3(grid), dim3(THREADS2), C::SMEM_BYTES, stream, map, a) != cudaSuccess) return SASSD_ERR_LAUNCH;
    return sassd_check_launch();
}

}  // namespace tma

extern "C" int sassd_conv2d_f16x3(const sassd_conv2d_desc* d, const void* in_split, const void* wpack,
                                  const float* scale, const float* shift, float* out_f32, void* out_split,
                                  sassd_stream_t stream_) {
    return sassd_conv2d_f16x3_occ(d, in_split, wpack, scale, shift, out_f32, out_split, nullptr, 0, nullptr, nullptr, stream_);
}

extern "C" int sassd_conv2d_f16x3_occ(const sassd_conv2d_desc* d, const void* in_split, const void* wpack,
                                      const float* scale, const float* shift, float* out_f32, void* out_split,
                                      const int32_t* tile_dist, int reach, const float* const_out, int32_t* counters,
                                      sassd_stream_t stream_) {
    if (tile_dist && (!const_out || reach < 0)) return SASSD_ERR_ARG;
    if (tile_dist) {
        // The constant-region rule is exact only while (a) the layer is within the range tile distances are recorded
        // for and (b) the zero-padding disturbance (reach-1 pixels deep) stays inside the outermost tile row / column,
        // the only tiles the kernel exempts - a thin partial edge tile would let it spill into a skipped tile.
        const int last_h = d ? d->H - (d->H - 1) / SASSD_CONV2D_TILE_H * SASSD_CONV2D_TILE_H : 0;
        const int last_w = d ? d->W - (d->W - 1) / SASSD_CONV2D_TILE_W * SASSD_CONV2D_TILE_W : 0;
        const int edge = last_h < last_w ? last_h : last_w;
        if (reach > SASSD_TILE_DIST_MAX || (edge < SASSD_CONV2D_TILE_H ? edge : SASSD_CONV2D_TILE_H) < reach - 1)
            return SASSD_ERR_UNSUPPORTED;
    }
    using namespace tma;
    if (!d || !in_split || !wpack || (!out_f32 && !out_split)) return SASSD_ERR_ARG;
    if (d->batch < 1 || d->H < 1 || d->W < 1 || d->cin < 1 || d->cout < 1 || d->cout > 256) return SASSD_ERR_ARG;
    if (!(d->taps == 9 || d->taps == 1) || (d->cin_stored % 64) != 0 || d->cin_stored < d->cin) return SASSD_ERR_ARG;
    if (out_split && ((d->out_split_ch % 8) != 0 || d->out_split_ch < 32)) return SASSD_ERR_ARG;
    if (out_f32 && (d->out_f32_stride % 4) != 0) return SASSD_ERR_ARG;
    EncodeTiledFn enc = get_encode();
    if (!enc) return SASSD_ERR_UNSUPPORTED;
    CUtensorMap map;
    // dims innermost first: channels, x, y, plane*batch ; fp16 elements
    cuuint64_t dims[4] = {(cuuint64_t)d->cin_stored, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)(2 * d->batch)};
    cuuint64_t strides[3] = {(cuuint64_t)d->cin_stored * 2, (cuuint64_t)d->W * d->cin_stored * 2,
                             (cuuint64_t)d->H * d->W * d->cin_stored * 2};
    cuuint32_t box[4] = {(cuuint32_t)BKC, (cuuint32_t)TILE_W, (cuuint32_t)TILE_H, 1u};
    cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
    CUresult rc = enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(in_split), dims, strides, box, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (rc != CUDA_SUCCESS) return SASSD_ERR_LAUNCH;
    Conv2dArgs a;
    a.wpack = wpack; a.scale = scale; a.shift = shift; a.out_f32 = out_f32; a.out_split = (__half*)out_split;
    a.batch = d->batch; a.H = d->H; a.W = d->W; a.cin = d->cin; a.cout = d->cout; a.taps = d->taps; a.relu = d->relu;
    a.out_f32_stride = d->out_f32_stride; a.out_split_ch = d->out_split_ch;
    a.tile_dist = tile_dist; a.reach = reach; a.cvec = const_out; a.counters = counters;
    a.tile_order = d->tile_order;
    a.nsplit = 1;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (d->cout <= 32) return launch2<32>(map, a, stream);
    if (d->cout <= 64) return launch2<64>(map, a, stream);
    if (d->cout <= 128) return launch2<128>(map, a, stream);
    // 128 < cout <= 256: two units per tile, each 128 output channels of the 256-wide weight pack
    a.nsplit = 2;
    return launch2<128>(map, a, stream);
}

// SparseConvTensor.dense() into the split BEV map: hi / lo*2048 fp16 planes [2,B,H,W,D*C] (channel d*C + c).
__global__ void sparse_to_bev_split_kernel(const float4* __restrict__ feat, const int4* __restrict__ coors,
                                           const int* __restrict__ d_rows, int rows_cap, int C4, int D, int H, int W,
                                           size_t plane, __half* __restrict__ bev, int* __restrict__ tile_dist) {
    const int rows = min(*d_rows, rows_cap);
    const long long total = (long long)rows * C4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i / C4), q = (int)(i % C4);
        const int4 c = __ldg(&coors[r]);
        const float4 v = __ldg(&feat[i]);
        uint32_t h0, h1, l0, l1;
        tc::split_f16x2(v.x, v.y, h0, l0);
        tc::split_f16x2(v.z, v.w, h1, l1);
        __half* dst = bev + ((((size_t)c.x * H + c.z) * W + c.w) * (size_t)(D * C4) + (size_t)c.y * C4 + q) * 4;
        *(uint2*)dst = make_uint2(h0, h1);
        *(uint2*)(dst + plane) = make_uint2(l0, l1);
        if (tile_dist && q == 0) sassd_mark_conv2d_tiles(tile_dist, c.x, c.z, c.w, H, W);
    }
}

extern "C" int sassd_sparse_to_bev_split(const float* feat, const int32_t* coors, const int32_t* d_rows, int rows_cap,
                                         int C, int D, int H, int W, int batch, void* bev_split, int32_t* tile_dist,
                                         sassd_stream_t stream_) {
    if (!feat || !coors || !d_rows || !bev_split || (C & 3) || batch < 1) return SASSD_ERR_ARG;
    if (rows_cap <= 0) return SASSD_OK;
    const size_t plane = (size_t)batch * H * W * D * C;
    sparse_to_bev_split_kernel<<<sassd_grid((long long)rows_cap * (C / 4), 256), 256, 0, (cudaStream_t)stream_>>>(
        (const float4*)feat, (const int4*)coors, d_rows, rows_cap, C / 4, D, H, W, plane, (__half*)bev_split, tile_dist);
    return sassd_check_launch();
}

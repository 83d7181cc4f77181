// Dense NHWC 3x3 / 1x1 convolution + folded BatchNorm + ReLU for the BEV neck and the heads
// (BEVNet cmn.py:233-282, SSDRotateHead ssd_rotate_head.py:218-231, PSWarpHead.convs :424-429),
// Hopper tensor cores (wgmma) on FP16x3, with the activation operand moved by TMA.
//
// Why a second tensor-core kernel: in gconv_tc.cu the A operand is gathered by producer warps
// (LDG -> split -> STS), nine times per element for a 3x3 conv.  Here
//   * activations live in HBM already split: two fp16 planes [2][B][H][W][C] (hi, lo*2048), written
//     once by the epilogue of the producing layer (or by the sparse->BEV scatter);
//   * a tile is an 8x16-pixel patch; a unit walks (tap column dx, 64-channel chunk) outer and the vertical taps dy
//     inner.  Per (dx, chunk) the A operand is ONE cp.async.bulk.tensor.4d halo box {64 ch, 16 x, 10 y, 1} per plane
//     at (y0-1, x0+dx) that all three dy taps read, at 2048-byte row offsets (a 1x1 conv: one column, an 8-row box) —
//     TMA writes it 128B-swizzled straight into the wgmma operand layout and zero-fills out-of-image pixels (= the
//     conv's zero padding);
//   * BN <= 64 (the PSWarp 3x3 256->28 conv, the head and PSWarp 1x1 convs): two rings, A stages (40 KB, released
//     after the box's last tap) and B stages (one (tap, chunk) of weights); no producer warps: warp 8 lane 0 issues
//     the TMA boxes (A hi, A lo) and the weight bulk copies, two consumer warpgroups (pixel rows 0-63 / 64-127 of the
//     tile) issue the MMAs and store the outputs from registers;
//   * BN = 128 (every layer with cout > 64): the operand roles are swapped.  The output channels are wgmma's M and the
//     tile's 128 pixels its N: consumer warpgroup wg owns channels 64 wg .. 64 wg + 63 of the unit and every pixel,
//     and issues m64n128k16 with the weights as A in registers and the halo box as B from shared memory.  The weights
//     are packed in wgmma's fragment order (sassd_conv2d_pack); one producer warp copies each chunk of them (32 KB)
//     with bulk copies into a two-stage ring, and the consumers move a chunk from the ring into registers one chunk
//     ahead of its MMAs and release the stage at once.  A producer warpgroup (setmaxnreg down to 40 registers, the
//     consumers up to 232) issues the boxes into a two-stage ring and the weights, and the epilogue transposes each
//     warpgroup's 64-channel x 128-pixel block through shared memory into 16-byte stores.
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
constexpr int kBgTile = 1 << 29;                // tile reference flag: the tile copies the layer's background map
constexpr int CONS_WARPS = CONS_THREADS / 32;   // 8
constexpr int W_LOAD = CONS_WARPS;

// The A operand of a (dx, chunk) step is one halo box per plane: TILE_H + 2 pixel rows (TILE_H for a 1x1 conv) of
// TILE_W pixels; the three vertical taps read it at row offsets 0, 1, 2, i.e. 2048-byte (swizzle-phase preserving) steps.
constexpr int A_ROWS = TILE_H + 2;
constexpr int A_PLANE_BYTES = A_ROWS * TILE_W * 128;    // 20 KB (hi) ; same for lo, right after it
constexpr int A_STAGE_BYTES = 2 * A_PLANE_BYTES;

// BN = 128 weight pack (sassd_conv2d_pack): per chunk q of a unit's walk, K step s (16 input channels) and block mb of
// 64 output channels, 128 threads x 32 bytes: thread t's wgmma A fragment, hi a0..a3 then lo a0..a3.  A unit's two
// blocks of a K step are contiguous: 8 KB per K step, 32 KB per chunk.
constexpr int FRAG_BLOCK_BYTES = 128 * 32;
constexpr int OUT_PITCH = 64 + 4;               // floats per pixel of the epilogue staging: conflict-free transposes

template <int BN>
struct Cfg2 {
    static constexpr bool RS = BN >= 128;                       // weights in registers (see the top of the file)
    static constexpr int THREADS = CONS_THREADS + (RS ? 128 : 32);
    static constexpr int A_STAGES = 2;
    static constexpr int B_TILE_BYTES = BN * 128;
    static constexpr int B_STAGE_BYTES = 2 * B_TILE_BYTES;     // one (tap, chunk): hi | lo; RS: one chunk of fragments
    static_assert(!RS || B_STAGE_BYTES == 4 * 2 * FRAG_BLOCK_BYTES, "an RS weight stage holds one chunk of a unit");
    static constexpr int B_STAGES = RS ? 2 : 6;
    static constexpr int OUT_BYTES = RS ? 2 * TILE_H * TILE_W * OUT_PITCH * 4 : 0;   // per warpgroup 128 px x 64 ch
    static constexpr int RING_BYTES = A_STAGES * A_STAGE_BYTES + B_STAGES * B_STAGE_BYTES + OUT_BYTES;
    // tile order (computed tiles first) when the map carries constant-region information: two verdict bits and a uint16
    // per tile, up to 16 frames of the 200 x 176 BEV grid (4400 tiles); the word keeps the tile index in 14 bits
    static constexpr int ORDER_CAP = 4608;
    static constexpr int SMEM_BYTES = RING_BYTES + 1024 + 256 + ORDER_CAP / 4 + ORDER_CAP * 2;
    static_assert(SMEM_BYTES <= 227 * 1024, "dynamic shared memory above the sm_90 limit");
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
    int* counters;        // optional [2]: += tiles computed (not stored or copied), += tiles (bench instrumentation)
    int tile_order;       // 1: computed tiles first, 0: round-robin
    int nsplit;           // work units per tile: 1, or 2 = each unit computes BN of the 2*BN output channels (the weight
                          // pack is the 2*BN-wide one)
    int* status;          // optional: SASSD_FLAG_F16_RANGE when a value stored into out_split overflows the split
};

// BN = 128 only, optional (see sassd_conv2d_desc): [B * tiles_y * tiles_x + 1] counters of the input map, written by
// the previous launch, and of this layer's output.  With in_ready the kernel starts without waiting for the previous
// grid and loads a unit's boxes once the tiles they read are ready.  A parameter of its own after the others: grown,
// Conv2dArgs moves the kernel's other parameters and costs the consumers of the kernel without counters a spill.
struct Ready {
    const int* in_ready;
    int* out_ready;
};

// Tile ready counters: every unit adds 2 / nsplit per warpgroup once its stores are done, so a tile's counter reaches
// kTileReady when all of its units have stored.  Word ntiles (after the tiles) counts the CTAs past their prologue.
constexpr int kTileReady = 4;
constexpr uint32_t kWaitCycles = 2000000000u;      // ~1 s at the H100's SM clocks: a wait past it is a bug, reported

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// After a barrier over the threads whose stores it publishes.
__device__ __forceinline__ void signal_ready(int* p, int v) {
    asm volatile("fence.acq_rel.gpu;\n\tred.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// Spins until *c >= target; false (and SASSD_FLAG_TILE_WAIT in the status word) once clock() is kWaitCycles past t0.
__device__ __forceinline__ bool wait_ready(const Conv2dArgs& p, const int* c, int target, uint32_t t0) {
    while (ld_acquire_gpu(c) < target) {
        if ((uint32_t)clock() - t0 > kWaitCycles) {
            if (p.status) atomicOr(p.status, SASSD_FLAG_TILE_WAIT);
            return false;
        }
        __nanosleep(64);
    }
    return true;
}
// The input tiles a unit of `tile` (b, ty, tx) reads: its halo box spans pixel rows y0 - halo .. y0 + TILE_H - 1 + halo
// and columns x0 - halo .. x0 + TILE_W - 1 + halo, i.e. the tiles ty - halo .. ty + halo, tx - halo .. tx + halo of
// frame b (halo = 1 <= TILE_H, TILE_W), clipped at the map edge, where TMA fills zeros.  Compact: it runs in the
// producer warpgroup's 40 registers.
__device__ __forceinline__ bool wait_input_tiles(const Conv2dArgs& p, const int* in_ready, int tile, int halo,
                                                 int tiles_y, int tiles_x) {
    const uint32_t t0 = (uint32_t)clock();
    const int ty = (tile / tiles_x) % tiles_y, tx = tile % tiles_x;
    for (int dy = -halo; dy <= halo; ++dy)
        for (int dx = -halo; dx <= halo; ++dx) {
            if (ty + dy < 0 || ty + dy >= tiles_y || tx + dx < 0 || tx + dx >= tiles_x) continue;
            if (!wait_ready(p, in_ready + tile + dy * tiles_x + dx, kTileReady, t0)) return false;
        }
    return true;
}

// Optional: the layer's outputs on an empty scene, batch 1 (same H, W, strides), copied into the far border tiles.
struct Background {
    const __half* split;
    const float* f32;
};

// How tile (ty, tx) at distance `dist` from the active cells is produced (see sassd_conv2d_f16x3_occ_bg in the header):
// 0 = computed; kConstTile = it sees a constant input and its output is p.cvec; kBgTile = it sees only inactive cells
// and the zero padding, so its output is the background map's at the same pixels.
__device__ __forceinline__ int tile_skip_flag(const Conv2dArgs& p, const Background& bg, int dist, int ty, int tx,
                                              int tiles_y, int tiles_x) {
    if (dist <= p.reach) return 0;
    if (p.reach < 2 || !(ty == 0 || ty == tiles_y - 1 || tx == 0 || tx == tiles_x - 1)) return kConstTile;
    return (bg.split || bg.f32) ? kBgTile : 0;      // the border sees the zero padding, which differs from cvec
}

// A unit of a background tile: channels [n_off, n_off + bn) of its pixels copied from the background map (batch 1) to
// frame b, split planes and fp32 alike, with 16-byte loads and stores by the nthreads consumer threads.  The same
// columns the register epilogue writes: those below out_split_ch / out_f32_stride.
__device__ __forceinline__ void copy_background_unit(const Conv2dArgs& p, const Background& bg, int b, int ty, int tx,
                                                     int n_off, int bn, int tid, int nthreads) {
    const size_t hw = (size_t)p.H * p.W;
    if (p.out_split) {
        const int vpp = min(bn, p.out_split_ch - n_off) >> 3;            // 16-byte vectors per pixel and plane
        const size_t bg_plane = hw * p.out_split_ch, plane = (size_t)p.batch * bg_plane;
        for (int i = tid; i < TILE_H * TILE_W * vpp; i += nthreads) {
            const int pix = i / vpp;
            const int y = ty * TILE_H + pix / TILE_W, x = tx * TILE_W + pix % TILE_W;
            if (y >= p.H || x >= p.W) continue;
            const size_t src = ((size_t)y * p.W + x) * p.out_split_ch + n_off + 8 * (i % vpp);
            const uint4 hi = __ldg((const uint4*)(bg.split + src));
            const uint4 lo = __ldg((const uint4*)(bg.split + bg_plane + src));
            __half* dst = p.out_split + (size_t)b * bg_plane + src;
            *(uint4*)dst = hi;
            *(uint4*)(dst + plane) = lo;
        }
    }
    if (p.out_f32) {
        const int vpp = min(bn, p.out_f32_stride - n_off) >> 2;
        for (int i = tid; i < TILE_H * TILE_W * vpp; i += nthreads) {
            const int pix = i / vpp;
            const int y = ty * TILE_H + pix / TILE_W, x = tx * TILE_W + pix % TILE_W;
            if (y >= p.H || x >= p.W) continue;
            const size_t src = ((size_t)y * p.W + x) * p.out_f32_stride + n_off + 4 * (i % vpp);
            *(float4*)(p.out_f32 + (size_t)b * hw * p.out_f32_stride + src) = __ldg((const float4*)(bg.f32 + src));
        }
    }
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
    F16Range ovf;
    ovf.add(lo.x); ovf.add(lo.y); ovf.add(lo.z); ovf.add(lo.w);
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
    report_f16_range(p.status, ovf.overflowed());
}

// Zeros in the stored channels [c0, out_split_ch) of a tile that lie past the columns of its units (c0 = nsplit * BN; a
// BN = 32 layer stores 64 channels), by nthreads threads: the next layer reads them through its 64-channel boxes, and
// the buffer may hold anything before the call.
__device__ __forceinline__ void zero_split_tail(const Conv2dArgs& p, int b, int ty, int tx, int c0, int tid,
                                                int nthreads) {
    if (!p.out_split || c0 >= p.out_split_ch) return;
    const int vpp = (p.out_split_ch - c0) >> 3;                        // 16-byte vectors per pixel and plane
    const size_t plane = (size_t)p.batch * p.H * p.W * p.out_split_ch;
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    for (int i = tid; i < TILE_H * TILE_W * vpp; i += nthreads) {
        const int pix = i / vpp;
        const int y = ty * TILE_H + pix / TILE_W, x = tx * TILE_W + pix % TILE_W;
        if (y >= p.H || x >= p.W) continue;
        __half* dst = p.out_split + (((size_t)b * p.H + y) * p.W + x) * p.out_split_ch + c0 + 8 * (i % vpp);
        *(uint4*)dst = zero;
        *(uint4*)(dst + plane) = zero;
    }
}

// One chunk (four K steps) of the BN = 128 split product with the weights in registers: w holds, per K step s,
// the hi fragment at w[8 s .. 8 s + 3] and the lo fragment at w[8 s + 4 .. 8 s + 7]; x_hi / x_lo are the pixels'
// K-major planes.  Same products and order per accumulator as mma_chunk_x3: small += wh*xl, small += wl*xh,
// big += wh*xh.
__device__ __forceinline__ void mma_chunk_x3_rs(float (&big)[64], float (&small)[64], const uint32_t (&w)[32],
                                                uint32_t x_hi, uint32_t x_lo) {
    const uint64_t dxh = make_desc(x_hi), dxl = make_desc(x_lo);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint64_t ko = 2ull * (uint64_t)k;
        const uint32_t wh[4] = {w[8 * k], w[8 * k + 1], w[8 * k + 2], w[8 * k + 3]};
        const uint32_t wl[4] = {w[8 * k + 4], w[8 * k + 5], w[8 * k + 6], w[8 * k + 7]};
        wgmma_rs_n128(small, wh, dxl + ko);
        wgmma_rs_n128(small, wl, dxh + ko);
        wgmma_rs_n128(big, wh, dxh + ko);
    }
}

// READY: the launch has tile ready counters (in_ready and / or out_ready, BN = 128 only); without them the kernel is
// compiled without their code.
template <int BN, bool READY>
__global__ void __launch_bounds__(Cfg2<BN>::THREADS, 1)
conv2d_tma_kernel(const __grid_constant__ CUtensorMap amap, const Conv2dArgs p, const Background bg, const Ready r) {
    using C = Cfg2<BN>;
    constexpr int A_STAGES = C::A_STAGES;
    extern __shared__ uint8_t smem_raw[];
    __shared__ int s_ncomp;       // computed tiles at the head of the tile order
    __shared__ int s_walk[6];     // see next_unit
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
    // A stages (halo boxes, hi | lo) at base; after them the B stages (BN <= 64: the weights of one (tap, chunk),
    // hi | lo; BN = 128: one chunk of the unit's weight fragments), then for BN = 128 the epilogue staging
    const uint32_t b_ring = base + A_STAGES * A_STAGE_BYTES;
    const uint32_t bar_base = base + C::RING_BYTES;
    auto a_full = [&](int s) { return bar_base + 8u * s; };
    auto a_empty = [&](int s) { return bar_base + 8u * (A_STAGES + s); };
    auto b_full = [&](int s) { return bar_base + 8u * (2 * A_STAGES + s); };
    auto b_empty = [&](int s) { return bar_base + 8u * (2 * A_STAGES + C::B_STAGES + s); };

    pdl_launch_dependents();      // the next layer may be scheduled as this grid's CTAs retire
    // warp index through a shuffle so that the compiler knows it is warp-uniform
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
    const int tiles_x = (p.W + TILE_W - 1) / TILE_W, tiles_y = (p.H + TILE_H - 1) / TILE_H;
    const int ntiles = p.batch * tiles_y * tiles_x;
    const int nsplit = p.nsplit, nunits = ntiles * nsplit;      // work unit k: tile k / nsplit, output channels (k % nsplit) * BN ...
    const int kchunks = (p.cin + BKC - 1) / BKC;
    const int nchunks = p.taps * kchunks;
    // A unit walks (dx, chunk) outer and dy inner: ncols = 3 (1) tap columns, each chunk's box serves nrows = 3 (1) taps
    const int ncols = p.taps == 9 ? 3 : 1, nrows = ncols, halo = ncols / 2;

    if (threadIdx.x == 0) {
        for (int s = 0; s < A_STAGES; ++s) { mbar_init(a_full(s), 1); mbar_init(a_empty(s), 2); }
        for (int s = 0; s < C::B_STAGES; ++s) { mbar_init(b_full(s), 1); mbar_init(b_empty(s), 2); }
        fence_barrier_init();
        asm volatile("prefetch.tensormap [%0];" ::"l"(&amap) : "memory");
        s_walk[0] = s_walk[1] = nunits;                 // round-robin; next_unit() with the tile order is set below
        s_walk[2] = s_walk[4] = nunits + blockIdx.x;
        s_walk[3] = 1;
        s_walk[5] = blockIdx.x;
    }
    __syncthreads();
    if (READY && r.in_ready) {
        // The producing layer may still be running; its units are waited for tile by tile before their boxes load.
        // The tile distances below were written before it started: reading them waits only until one of its CTAs
        // has passed this point, which orders them (and the zeroed counters) before everything this grid reads.
        if (threadIdx.x == 0) wait_ready(p, r.in_ready + ntiles, 1, (uint32_t)clock());
        __syncthreads();
    } else {
        pdl_wait();               // the producing layer has completed; nothing above touched global data
    }
    if (READY && r.out_ready && threadIdx.x == 0) signal_ready(r.out_ready + ntiles, 1);

    // With constant-region information most tiles only store a constant or copy the background.  Static round-robin
    // leaves some CTAs with two computed tiles and others with none (on the 11-tile-wide BEV grid a stride of 132 units
    // is 6 tile rows: a CTA stays in one tile column); with tile_order = 1 (for maps of up to ORDER_CAP tiles, above it
    // round-robin with per-tile distance loads) every CTA builds the same order - computed tiles first, stored and copied
    // tiles after - and all roles walk it as next_unit() deals it.  Round-robin is the default: with several steps in
    // flight the SMs that only store are what the other frames' kernels run on.
    uint32_t* verdict = (uint32_t*)(base_ptr + C::RING_BYTES + 256);   // [2][ORDER_CAP / 32]: constant, background bits
    uint16_t* order = (uint16_t*)(verdict + 2 * (C::ORDER_CAP / 32));
    const bool small_map = p.tile_dist != nullptr && ntiles <= C::ORDER_CAP;
    const bool use_order = p.tile_order && small_map;
    // For maps of up to ORDER_CAP tiles the CTA fetches every tile's distance once (one memory latency per four 32-tile
    // slots and warp instead of one per tile and role) and keeps the verdicts as order[k] bit 15 (constant) and bit 14
    // (background).
    if (small_map) {
        const int nslots = (ntiles + 31) / 32;
#pragma unroll 1
        for (int i0 = 4 * warp; i0 < nslots; i0 += 4 * (C::THREADS / 32)) {
            int dist[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int t = (i0 + e) * 32 + lane;
                dist[e] = t < ntiles ? __ldg(&p.tile_dist[t]) : 0;
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int t = (i0 + e) * 32 + lane;
                const int f = t < ntiles ? tile_skip_flag(p, bg, dist[e], (t / tiles_x) % tiles_y, t % tiles_x, tiles_y,
                                                          tiles_x) : 0;
                const uint32_t cst = __ballot_sync(0xffffffffu, f == kConstTile);
                const uint32_t bgm = __ballot_sync(0xffffffffu, f == kBgTile);
                if (lane == 0 && i0 + e < nslots) {
                    verdict[i0 + e] = cst;
                    verdict[C::ORDER_CAP / 32 + i0 + e] = bgm;
                }
            }
        }
        __syncthreads();
        if (warp == 0) {
            auto word = [&](int t, uint32_t cst, uint32_t bgm) {
                return (uint16_t)(t | (((cst >> lane) & 1u) ? 0x8000 : 0) | (((bgm >> lane) & 1u) ? 0x4000 : 0));
            };
            if (use_order) {
                int n = 0;
                for (int pass = 0; pass < 2; ++pass) {
#pragma unroll 1
                    for (int i = 0; i < nslots; ++i) {
                        const int t = i * 32 + lane;
                        const uint32_t cst = verdict[i], bgm = verdict[C::ORDER_CAP / 32 + i];
                        const bool skip = ((cst | bgm) >> lane) & 1u;
                        const bool take = t < ntiles && (skip == (pass == 1));
                        const uint32_t m = __ballot_sync(0xffffffffu, take);
                        if (take) order[n + __popc(m & ((1u << lane) - 1u))] = word(t, cst, bgm);
                        n += __popc(m);
                    }
                    if (pass == 0 && lane == 0) s_ncomp = n;
                }
                if (lane == 0) {
                    constexpr int kTailAbsorb = 8;
                    const int G = gridDim.x, c = blockIdx.x;
                    const int ucomp = s_ncomp * nsplit;
                    const int heavy = ucomp % G, light = G - heavy;
                    const int absorb = heavy ? min(nunits - ucomp, kTailAbsorb * light) : 0;
                    const int s2 = ucomp + c - heavy, s3 = ucomp + absorb + c;      // this CTA's first unit of each tail part
                    const int first_tail = (c >= heavy && s2 < ucomp + absorb) ? s2 : s3;
                    s_walk[0] = ucomp;
                    s_walk[1] = ucomp + absorb;
                    s_walk[2] = first_tail;
                    s_walk[3] = light;
                    s_walk[4] = s3;
                    s_walk[5] = c < ucomp ? c : first_tail;
                }
            } else {
#pragma unroll 1
                for (int i = 0; i < nslots; ++i) {
                    const int t = i * 32 + lane;
                    if (t < ntiles) order[t] = word(t, verdict[i], verdict[C::ORDER_CAP / 32 + i]);
                }
            }
        }
        __syncthreads();
    }
    // The units a CTA walks: s_walk[5], then next_unit(k) while below nunits.  Without the tile order: c, c + G, ...
    // (c = blockIdx.x, G = gridDim.x).  With it, the ucomp computed units go round-robin the same way, which leaves
    // `heavy` = ucomp % G CTAs with one more of them than the others; the stored and copied units after them go first to
    // the other CTAs, up to kTailAbsorb each (a store or copy takes a small fraction of a computed unit's time), and
    // round-robin over every CTA beyond that.  So the CTAs that compute most do not also store.  The walk lives in
    // shared memory: the BN = 128 consumers have no register to spare across their MMA loop.
    auto next_unit = [&](int k) -> int {
        if (k < s_walk[0]) { k += gridDim.x; return k < s_walk[0] ? k : s_walk[2]; }
        if (k < s_walk[1]) { k += s_walk[3]; return k < s_walk[1] ? k : s_walk[4]; }
        return k + gridDim.x;
    };
    // tile_ref(k): the k-th tile in walking order, | kConstTile when it only stores the layer's constant, | kBgTile when
    // it copies the background
    auto tile_ref = [&](int k) -> int {
        if (small_map) { const int v = order[k]; return (v & 0x3fff) | ((v & 0xc000) << 15); }
        if (!p.tile_dist) return k;
        return k | tile_skip_flag(p, bg, __ldg(&p.tile_dist[k]), (k / tiles_x) % tiles_y, k % tiles_x, tiles_y, tiles_x);
    };

    if (warp >= W_LOAD) {
        if constexpr (C::RS) {
            setmaxnreg_dec<40>();
            if (warp == W_LOAD + 1 && lane == 0) {
                // The weights of every computed unit, chunk by chunk in the order of the walk (the pack's): per K step
                // the unit's two blocks, 8 KB contiguous in the pack.
                constexpr uint32_t kStep = 2 * FRAG_BLOCK_BYTES;
                int b_stage = 0;
                uint32_t b_phase = 0;
                for (int k = s_walk[5]; k < nunits; k = next_unit(k)) {
                    if (tile_ref(k / nsplit) & (kConstTile | kBgTile)) continue;
                    const uint8_t* src = (const uint8_t*)p.wpack + (size_t)(k % nsplit) * kStep;
                    for (int q = 0; q < nchunks; ++q) {
                        mbar_wait(b_empty(b_stage), b_phase ^ 1u);
                        mbar_expect_tx(b_full(b_stage), C::B_STAGE_BYTES);
                        const uint32_t dst = b_ring + b_stage * C::B_STAGE_BYTES;
#pragma unroll 1
                        for (int s = 0; s < 4; ++s, src += (size_t)nsplit * kStep)
                            bulk_g2s(dst + s * kStep, src, kStep, b_full(b_stage));
                        if (++b_stage == C::B_STAGES) { b_stage = 0; b_phase ^= 1u; }
                    }
                }
            }
            if (warp != W_LOAD) return;
        }
        if (lane == 0) {
            int a_stage = 0, b_stage = 0;
            uint32_t a_phase = 0, b_phase = 0;
            // one box per plane and (dx, chunk): rows y0 - halo .. y0 + TILE_H - 1 + halo (the TMA box height of the map)
            const uint32_t a_bytes = 2u * (TILE_H + 2 * halo) * TILE_W * 128;
            bool waiting = READY && r.in_ready != nullptr;     // false after a timed-out wait: the status word reports it
            for (int k = s_walk[5]; k < nunits; k = next_unit(k)) {
                const int ref = tile_ref(k / nsplit), half = k % nsplit;
                if (ref & (kConstTile | kBgTile)) continue;                             // nothing to load
                const int tile = ref;
                const int b = tile / (tiles_y * tiles_x);
                const int ty = (tile / tiles_x) % tiles_y, tx = tile % tiles_x;
                const int y0 = ty * TILE_H, x0 = tx * TILE_W;
                if (READY && r.in_ready) {
                    if (waiting) waiting = wait_input_tiles(p, r.in_ready, tile, halo, tiles_y, tiles_x);
                    // the tiles were stored through the generic proxy on other SMs; the boxes read them through TMA
                    asm volatile("fence.proxy.async.global;" ::: "memory");
                }
                for (int col = 0; col < ncols; ++col) {
                    const int dx = col - halo;
                    for (int kc = 0; kc < kchunks; ++kc) {
                        mbar_wait(a_empty(a_stage), a_phase ^ 1u);
                        const uint32_t a_hi = base + a_stage * A_STAGE_BYTES;
                        mbar_expect_tx(a_full(a_stage), a_bytes);
                        // coordinates innermost first: {channel, x, y, plane*B + b}; out-of-image pixels arrive as zeros
                        tma_load_4d(a_hi, &amap, kc * BKC, x0 + dx, y0 - halo, b, a_full(a_stage));
                        tma_load_4d(a_hi + A_PLANE_BYTES, &amap, kc * BKC, x0 + dx, y0 - halo, p.batch + b, a_full(a_stage));
                        if (++a_stage == A_STAGES) { a_stage = 0; a_phase ^= 1u; }
                        if constexpr (!C::RS) {                  // BN = 128: warp W_LOAD + 1 copies the weights
                            for (int row = 0; row < nrows; ++row) {
                                const int t = row * ncols + col;                            // tap (dy + 1) * 3 + dx + 1
                                mbar_wait(b_empty(b_stage), b_phase ^ 1u);
                                const uint32_t b_dst = b_ring + b_stage * C::B_STAGE_BYTES;
                                mbar_expect_tx(b_full(b_stage), C::B_STAGE_BYTES);
                                // pack: per (tap, chunk) [hi | lo], each nsplit * BN rows of 128 bytes; this unit's BN rows
                                const uint8_t* src = (const uint8_t*)p.wpack +
                                                     (size_t)(t * kchunks + kc) * (size_t)(2 * nsplit) * C::B_TILE_BYTES +
                                                     (size_t)half * C::B_TILE_BYTES;
                                constexpr uint32_t kPiece = (C::B_TILE_BYTES >= 8192) ? 8192u : (uint32_t)C::B_TILE_BYTES;
#pragma unroll 1
                                for (int part = 0; part < 2; ++part)
#pragma unroll 1
                                    for (uint32_t o = 0; o < (uint32_t)C::B_TILE_BYTES; o += kPiece)
                                        bulk_g2s(b_dst + part * C::B_TILE_BYTES + o,
                                                 src + (size_t)part * nsplit * C::B_TILE_BYTES + o, kPiece, b_full(b_stage));
                                if (++b_stage == C::B_STAGES) { b_stage = 0; b_phase ^= 1u; }
                            }
                        }
                    }
                }
            }
        }
        // The stored channels past the units' columns of every tile this CTA walks (computed, stored or copied alike):
        // zeros, written by this warp while the consumers finish their MMAs (on the consumers' side the stores' address
        // arithmetic would be hoisted across the accumulators).
        if (p.out_split && nsplit * BN < p.out_split_ch) {
            __syncwarp();
            for (int k = s_walk[5]; k < nunits; k = next_unit(k)) {
                if (k % nsplit != nsplit - 1) continue;
                const int tile = tile_ref(k / nsplit) & ~(kConstTile | kBgTile);
                zero_split_tail(p, tile / (tiles_y * tiles_x), (tile / tiles_x) % tiles_y, tile % tiles_x, nsplit * BN,
                                lane, 32);
            }
        }
    } else {
        // ============ consumers: warpgroup wg owns pixel rows 64 wg .. 64 wg + 63 of the tile (BN <= 64) or ============
        // ============ output channels 64 wg .. 64 wg + 63 of the unit (BN = 128)                            ============
        if constexpr (C::RS) setmaxnreg_inc<232>();
        const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
        const int rl0 = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);        // tile rows rl0 and rl0 + 8 (= pixel py * 16 + px)
        const size_t plane = (size_t)p.batch * p.H * p.W * p.out_split_ch;
        float big[BN / 2], small[BN / 2];
        int a_stage = 0, b_stage = 0;
        uint32_t a_phase = 0, b_phase = 0;
        int computed = 0;
        // A unit of tile (b, ty, tx) has stored everything this warpgroup writes of it: publish the warpgroup's share.
        auto unit_stored = [&](int b, int ty, int tx) {
            if constexpr (READY) {
                if (r.out_ready) {
                    // everything from the thread index and the parameters: no register is kept across the MMA loop
                    named_bar_sync(1 + (threadIdx.x >> 7), 128);
                    const int ntx = (p.W + TILE_W - 1) / TILE_W, nty = (p.H + TILE_H - 1) / TILE_H;
                    if ((threadIdx.x & 127) == 0) signal_ready(r.out_ready + (b * nty + ty) * ntx + tx, 2 / p.nsplit);
                }
            }
        };
        for (int k = s_walk[5]; k < nunits; k = next_unit(k)) {
            const int ref = tile_ref(k / nsplit), n_off = (k % nsplit) * BN;
            const int tile = ref & ~(kConstTile | kBgTile);
            const bool const_tile = (ref & kConstTile) != 0;
            const int b = tile / (tiles_y * tiles_x);
            const int ty = (tile / tiles_x) % tiles_y, tx = tile % tiles_x;
            if (ref & kBgTile) continue;                                  // copied after this loop
            if (const_tile) {                                               // no MMAs run for this tile
                const int ncols = min(BN, p.out_split_ch - n_off);
                if (p.out_split && !p.out_f32 && (ncols == 64 || ncols == 128 || ncols == 256)) {
                    store_constant_unit<CONS_WARPS>(p, b, ty, tx, n_off, ncols, warp, lane);
                    if constexpr (READY) goto stored;      // one signal site: a second costs the consumers a spill
                    continue;
                }
            } else {
                if (k % nsplit == 0) ++computed;
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) { big[i] = 0.f; small[i] = 0.f; }
                // stages the previous chunk's MMAs read: released once they are known complete (prev_a only after
                // the last of the box's nrows taps)
                int prev_b = -1, prev_a = -1, row = 0;
                if constexpr (C::RS) {
                    // The next chunk's fragments from the weight ring: per K step s this warpgroup's block at
                    // 8 KB s + 4 KB wg, thread t's 32 bytes (hi | lo) in it.  Threads with (t / 4) odd read their lo
                    // half first, so that each 8-thread phase of a 16-byte load covers all 32 banks.  The stage is
                    // released as soon as every thread of the warpgroup holds its fragments.
                    auto load_w = [&](uint32_t (&w)[32]) {
                        mbar_wait(b_full(b_stage), b_phase);
                        const uint32_t sw = (t & 4) * 4u;
                        const uint32_t src = b_ring + b_stage * C::B_STAGE_BYTES + wg * FRAG_BLOCK_BYTES + t * 32;
#pragma unroll
                        for (int s = 0; s < 4; ++s) {
                            const uint4 x = lds_v4(src + s * 2 * FRAG_BLOCK_BYTES + sw);
                            const uint4 y = lds_v4(src + s * 2 * FRAG_BLOCK_BYTES + (sw ^ 16u));
                            const uint4 h = sw ? y : x, l = sw ? x : y;
                            w[8 * s] = h.x; w[8 * s + 1] = h.y; w[8 * s + 2] = h.z; w[8 * s + 3] = h.w;
                            w[8 * s + 4] = l.x; w[8 * s + 5] = l.y; w[8 * s + 6] = l.z; w[8 * s + 7] = l.w;
                        }
                        named_bar_sync(3 + wg, 128);
                        if (t == 0) mbar_arrive(b_empty(b_stage));
                        if (++b_stage == C::B_STAGES) { b_stage = 0; b_phase ^= 1u; }
                    };
                    // Chunk ch on the fragments in w; the next chunk's go into w_next once the MMAs that read them
                    // (chunk ch - 1) are complete.
                    auto chunk = [&](uint32_t (&w)[32], uint32_t (&w_next)[32], int ch) {
                        if (row == 0) mbar_wait(a_full(a_stage), a_phase);
                        const uint32_t xh = base + a_stage * A_STAGE_BYTES + (uint32_t)row * (TILE_W * 128u);
                        wgmma_fence();
                        mma_chunk_x3_rs(big, small, w, xh, xh + A_PLANE_BYTES);
                        wgmma_commit();
                        wgmma_wait<1>();
                        fence_regs<32>(w_next);
                        if (t == 0 && prev_a >= 0) mbar_arrive(a_empty(prev_a));
                        if (ch + 1 < nchunks) load_w(w_next);
                        prev_a = -1;
                        if (++row == nrows) {
                            row = 0;
                            prev_a = a_stage;
                            if (++a_stage == A_STAGES) { a_stage = 0; a_phase ^= 1u; }
                        }
                    };
                    uint32_t wa[32], wb[32];
                    load_w(wa);
                    for (int ch = 0; ch < nchunks; ch += 2) {
                        chunk(wa, wb, ch);
                        if (ch + 1 == nchunks) break;
                        chunk(wb, wa, ch + 1);
                    }
                    wgmma_wait<0>();
                    fence_regs<32>(wa);
                    fence_regs<32>(wb);
                } else {
                    for (int ch = 0; ch < nchunks; ++ch) {
                        if (row == 0) mbar_wait(a_full(a_stage), a_phase);
                        mbar_wait(b_full(b_stage), b_phase);
                        // tap row `row` of this warpgroup's 4 pixel rows: box rows row + 4 wg .. row + 4 wg + 3
                        const uint32_t ah = base + a_stage * A_STAGE_BYTES + (uint32_t)(row * TILE_W + wg * 64) * 128u;
                        const uint32_t bh = b_ring + b_stage * C::B_STAGE_BYTES;
                        wgmma_fence();
                        mma_chunk_x3<1, BN>(big, small, ah, ah + A_PLANE_BYTES, bh, bh + C::B_TILE_BYTES);
                        wgmma_commit();
                        wgmma_wait<1>();            // the previous chunk's MMAs have read their stages
                        if (t == 0) {
                            if (prev_b >= 0) mbar_arrive(b_empty(prev_b));
                            if (prev_a >= 0) mbar_arrive(a_empty(prev_a));
                        }
                        prev_b = b_stage;
                        if (++b_stage == C::B_STAGES) { b_stage = 0; b_phase ^= 1u; }
                        prev_a = -1;
                        if (++row == nrows) {
                            row = 0;
                            prev_a = a_stage;
                            if (++a_stage == A_STAGES) { a_stage = 0; a_phase ^= 1u; }
                        }
                    }
                }
                wgmma_wait<0>();
                fence_regs<BN / 2>(big);
                fence_regs<BN / 2>(small);
                if (t == 0) {
                    if (prev_b >= 0) mbar_arrive(b_empty(prev_b));
                    if (prev_a >= 0) mbar_arrive(a_empty(prev_a));
                }
            }
            if constexpr (C::RS) {
                // Epilogue through shared memory: thread t holds channels m0, m0 + 8 of the warpgroup's 64 at pixels
                // 8 j + 2 (t % 4) + e; folded BN + ReLU (or the layer constant) into the warpgroup's staging block
                // [pixel][OUT_PITCH], then whole pixels out with 16-byte fp32 and / or split-plane stores.
                float* stage = (float*)(base_ptr + A_STAGES * A_STAGE_BYTES + C::B_STAGES * C::B_STAGE_BYTES) +
                               wg * (TILE_H * TILE_W * OUT_PITCH);
                const int m0 = 16 * (t >> 5) + ((t & 31) >> 2), c_wg = n_off + 64 * wg;
                float cv[2], sc[2], sh[2];
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int n = c_wg + m0 + 8 * i;
                    cv[i] = const_tile && n < p.cout ? __ldg(&p.cvec[n]) : 0.f;
                    sc[i] = p.scale && n < p.cout ? __ldg(&p.scale[n]) : 1.f;
                    sh[i] = p.shift && n < p.cout ? __ldg(&p.shift[n]) : 0.f;
                }
                named_bar_sync(1 + wg, 128);        // the warpgroup's read-back of the previous unit is done
#pragma unroll
                for (int j = 0; j < 16; ++j)
#pragma unroll
                    for (int i = 0; i < 2; ++i)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            float o = cv[i];
                            if (!const_tile) {
                                o = fmaf(__fadd_rn(big[4 * j + 2 * i + e], small[4 * j + 2 * i + e] * (1.f / kF16LoScale)),
                                         sc[i], sh[i]);
                                if (p.relu) o = sassd_relu(o);
                                if (c_wg + m0 + 8 * i >= p.cout) o = 0.f;
                            }
                            stage[(8 * j + 2 * (t & 3) + e) * OUT_PITCH + m0 + 8 * i] = o;
                        }
                named_bar_sync(1 + wg, 128);
                if (p.out_f32) {
                    for (int v = t; v < TILE_H * TILE_W * 16; v += 128) {
                        const int pix = v >> 4, c = 4 * (v & 15), n = c_wg + c;
                        const int y = ty * TILE_H + pix / TILE_W, x = tx * TILE_W + pix % TILE_W;
                        if (n >= p.out_f32_stride || y >= p.H || x >= p.W) continue;
                        *(float4*)(p.out_f32 + (((size_t)b * p.H + y) * p.W + x) * p.out_f32_stride + n) =
                            *(const float4*)(stage + pix * OUT_PITCH + c);
                    }
                }
                if (p.out_split) {
                    F16Range ovf;             // one vote per unit: no register lives across the MMA loop for it
                    for (int v = t; v < TILE_H * TILE_W * 8; v += 128) {
                        const int pix = v >> 3, c = 8 * (v & 7), n = c_wg + c;
                        const int y = ty * TILE_H + pix / TILE_W, x = tx * TILE_W + pix % TILE_W;
                        if (n >= p.out_split_ch || y >= p.H || x >= p.W) continue;
                        const float4 f0 = *(const float4*)(stage + pix * OUT_PITCH + c);
                        const float4 f1 = *(const float4*)(stage + pix * OUT_PITCH + c + 4);
                        uint4 hi, lo;
                        split_f16x2(f0.x, f0.y, hi.x, lo.x);
                        split_f16x2(f0.z, f0.w, hi.y, lo.y);
                        split_f16x2(f1.x, f1.y, hi.z, lo.z);
                        split_f16x2(f1.z, f1.w, hi.w, lo.w);
                        ovf.add(lo.x); ovf.add(lo.y); ovf.add(lo.z); ovf.add(lo.w);
                        __half* dst = p.out_split + (((size_t)b * p.H + y) * p.W + x) * p.out_split_ch + n;
                        *(uint4*)dst = hi;
                        *(uint4*)(dst + plane) = lo;
                    }
                    report_f16_range(p.status, ovf.overflowed());
                }
            } else {
                // epilogue from registers: folded BN + ReLU (or the layer constant), fp32 and / or split-plane stores
                F16Range ovf;
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
                            if (p.relu) { o0 = sassd_relu(o0); o1 = sassd_relu(o1); }
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
                            ovf.add(l);
                            __half* dst = p.out_split + pix * p.out_split_ch + n;
                            *(uint32_t*)dst = h;
                            *(uint32_t*)(dst + plane) = l;
                        }
                    }
                }
                report_f16_range(p.status, ovf.overflowed());
            }
        stored:
            unit_stored(b, ty, tx);
        }
        // Background tiles in a pass of their own: interleaved with the MMA units, the copy's address arithmetic is
        // hoisted across the accumulators and spills them.
        if (bg.split || bg.f32) {
            for (int k = s_walk[5]; k < nunits; k = next_unit(k)) {
                const int ref = tile_ref(k / nsplit);
                if (!(ref & kBgTile)) continue;
                const int tile = ref & ~kBgTile;
                copy_background_unit(p, bg, tile / (tiles_y * tiles_x), (tile / tiles_x) % tiles_y, tile % tiles_x,
                                     (k % nsplit) * BN, BN, threadIdx.x, CONS_THREADS);
                if constexpr (READY) unit_stored(tile / (tiles_y * tiles_x), (tile / tiles_x) % tiles_y, tile % tiles_x);
            }
        }
        if (p.counters && threadIdx.x == 0) {
            if (computed) atomicAdd(&p.counters[0], computed);
            if (blockIdx.x == 0) atomicAdd(&p.counters[1], ntiles);
        }
        // Without the wait at the start, this grid could complete before the producing layer.  Waiting here keeps
        // "this layer complete" implying "every earlier layer complete", which every launch after the chain relies on
        // (a grid completes only when all of its threads have exited, so the consumer threads' wait suffices).
        if (READY && r.in_ready) pdl_wait();
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

template <int BN, bool READY = false>
static int launch2(const CUtensorMap& map, const Conv2dArgs& a, const Background& bg, const Ready& r,
                   cudaStream_t stream) {
    using C = Cfg2<BN>;
    auto kern = conv2d_tma_kernel<BN, READY>;
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES) != cudaSuccess)
            return SASSD_ERR_LAUNCH;
        configured = true;
    }
    const int units = a.batch * sassd_div_up(a.H, TILE_H) * sassd_div_up(a.W, TILE_W) * a.nsplit;
    const int grid = units < sassd_num_sms() ? units : sassd_num_sms();
    if (launch_pdl(kern, dim3(grid), dim3(C::THREADS), C::SMEM_BYTES, stream, map, a, bg, r) != cudaSuccess)
        return SASSD_ERR_LAUNCH;
    return sassd_check_launch();
}

// The BN = 128 weight pack, W [taps, cin, cout] fp32 -> f16x2 words, one thread per word.  Chunk q of a unit's walk
// ((dx, chunk) outer, dy inner: q = (col * kchunks + kc) * nrows + row, tap row * ncols + col), K step s, block mb of
// 64 output channels and thread t hold hi a0..a3 then lo a0..a3, fragment register a (0..3) being output channel
// 64 mb + 16 (t / 32) + (t % 32) / 4 + 8 (a & 1) at input channels 64 kc + 16 s + 2 (t % 4) + 8 (a >> 1) + {0, 1}.
__global__ void conv2d_pack_kernel(const float* __restrict__ w, int taps, int cin, int cout, int nblk,
                                   uint32_t* __restrict__ out) {
    const int kchunks = (cin + BKC - 1) / BKC, ncols = taps == 9 ? 3 : 1, nrows = ncols;
    const long long total = (long long)taps * kchunks * 4 * nblk * (FRAG_BLOCK_BYTES / 4);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int word = (int)(i % 8), t = (int)((i / 8) % 128);
        long long r = i / (FRAG_BLOCK_BYTES / 4);
        const int mb = (int)(r % nblk);
        r /= nblk;
        const int s = (int)(r % 4), q = (int)(r / 4);
        const int row = q % nrows, kc = (q / nrows) % kchunks, col = q / (nrows * kchunks);
        const int tap = row * ncols + col, a = word % 4, lane = t % 32;
        const int n = 64 * mb + 16 * (t / 32) + lane / 4 + 8 * (a & 1);
        const int k = kc * BKC + 16 * s + 2 * (lane % 4) + 8 * (a >> 1);
        float hi[2], lo[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const float v = (k + e < cin && n < cout) ? w[((size_t)tap * cin + k + e) * cout + n] : 0.f;
            split_f16(v, hi[e], lo[e]);
        }
        const __half2 h = word < 4 ? __floats2half2_rn(hi[0], hi[1]) : __floats2half2_rn(lo[0], lo[1]);
        out[i] = *reinterpret_cast<const uint32_t*>(&h);
    }
}

}  // namespace tma

extern "C" int sassd_pdl_enabled(void) { return tc::pdl_enabled() ? 1 : 0; }

extern "C" size_t sassd_conv2d_pack_bytes(int taps, int cin, int cout) {
    if (!(taps == 9 || taps == 1) || cin < 1 || cout < 1 || cout > 256) return 0;
    if (cout <= 64) return sassd_gconv_pack_bytes(taps, cin, cout, SASSD_PREC_F16X3);
    return (size_t)taps * ((cin + tma::BKC - 1) / tma::BKC) * 4 * (cout <= 128 ? 2 : 4) * tma::FRAG_BLOCK_BYTES;
}

extern "C" int sassd_conv2d_pack(const float* weight, int taps, int cin, int cout, void* packed,
                                 sassd_stream_t stream_) {
    if (!weight || !packed || sassd_conv2d_pack_bytes(taps, cin, cout) == 0) return SASSD_ERR_ARG;
    if (cout <= 64) return sassd_gconv_pack(weight, taps, cin, cout, SASSD_PREC_F16X3, packed, stream_);
    const long long words = (long long)sassd_conv2d_pack_bytes(taps, cin, cout) / 4;
    tma::conv2d_pack_kernel<<<sassd_grid(words, 256), 256, 0, (cudaStream_t)stream_>>>(
        weight, taps, cin, cout, cout <= 128 ? 2 : 4, (uint32_t*)packed);
    return sassd_check_launch();
}

extern "C" int sassd_conv2d_f16x3(const sassd_conv2d_desc* d, const void* in_split, const void* wpack,
                                  const float* scale, const float* shift, float* out_f32, void* out_split,
                                  sassd_stream_t stream_) {
    return sassd_conv2d_f16x3_occ_bg_status(d, in_split, wpack, scale, shift, out_f32, out_split, nullptr, 0, nullptr,
                                            nullptr, nullptr, nullptr, nullptr, stream_);
}

extern "C" int sassd_conv2d_f16x3_occ(const sassd_conv2d_desc* d, const void* in_split, const void* wpack,
                                      const float* scale, const float* shift, float* out_f32, void* out_split,
                                      const int32_t* tile_dist, int reach, const float* const_out, int32_t* counters,
                                      sassd_stream_t stream_) {
    return sassd_conv2d_f16x3_occ_bg_status(d, in_split, wpack, scale, shift, out_f32, out_split, tile_dist, reach,
                                            const_out, nullptr, nullptr, counters, nullptr, stream_);
}

extern "C" int sassd_conv2d_f16x3_occ_bg(const sassd_conv2d_desc* d, const void* in_split, const void* wpack,
                                         const float* scale, const float* shift, float* out_f32, void* out_split,
                                         const int32_t* tile_dist, int reach, const float* const_out,
                                         const void* bg_split, const float* bg_f32, int32_t* counters,
                                         sassd_stream_t stream_) {
    return sassd_conv2d_f16x3_occ_bg_status(d, in_split, wpack, scale, shift, out_f32, out_split, tile_dist, reach,
                                            const_out, bg_split, bg_f32, counters, nullptr, stream_);
}

extern "C" int sassd_conv2d_f16x3_occ_bg_status(const sassd_conv2d_desc* d, const void* in_split, const void* wpack,
                                                const float* scale, const float* shift, float* out_f32,
                                                void* out_split, const int32_t* tile_dist, int reach,
                                                const float* const_out, const void* bg_split, const float* bg_f32,
                                                int32_t* counters, int32_t* d_status, sassd_stream_t stream_) {
    if (tile_dist && (!const_out || reach < 0)) return SASSD_ERR_ARG;
    // a background must hold every output the layer writes
    if ((bg_split || bg_f32) && ((out_split && !bg_split) || (out_f32 && !bg_f32))) return SASSD_ERR_ARG;
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
    // ready counters: BN = 128 launches only, without a zero tail (zero_split_tail's stores are not counted: every
    // stored channel must belong to a unit, out_split_ch <= nsplit * 128), and a timed-out wait needs the status word
    // to report it
    if ((d->in_ready || d->out_ready) &&
        (d->cout <= 64 || (out_split && d->out_split_ch > (d->cout > 128 ? 256 : 128))))
        return SASSD_ERR_ARG;
    if (d->in_ready && !d_status) return SASSD_ERR_ARG;
    EncodeTiledFn enc = get_encode();
    if (!enc) return SASSD_ERR_UNSUPPORTED;
    CUtensorMap map;
    // dims innermost first: channels, x, y, plane*batch ; fp16 elements
    cuuint64_t dims[4] = {(cuuint64_t)d->cin_stored, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)(2 * d->batch)};
    cuuint64_t strides[3] = {(cuuint64_t)d->cin_stored * 2, (cuuint64_t)d->W * d->cin_stored * 2,
                             (cuuint64_t)d->H * d->W * d->cin_stored * 2};
    // one box holds every row the tile's vertical taps read: the tile and a halo row above and below (3x3)
    cuuint32_t box[4] = {(cuuint32_t)BKC, (cuuint32_t)TILE_W, (cuuint32_t)(d->taps == 9 ? A_ROWS : TILE_H), 1u};
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
    a.status = d_status;
    const Ready r = {d->in_ready, d->out_ready};
    const Background bg = {out_split ? (const __half*)bg_split : nullptr, out_f32 ? bg_f32 : nullptr};
    cudaStream_t stream = (cudaStream_t)stream_;
    if (d->cout <= 32) return launch2<32>(map, a, bg, r, stream);
    if (d->cout <= 64) return launch2<64>(map, a, bg, r, stream);
    const bool ready = r.in_ready || r.out_ready;
    if (d->cout <= 128) return ready ? launch2<128, true>(map, a, bg, r, stream) : launch2<128>(map, a, bg, r, stream);
    // 128 < cout <= 256: two units per tile, each 128 output channels of the 256-wide weight pack
    a.nsplit = 2;
    return ready ? launch2<128, true>(map, a, bg, r, stream) : launch2<128>(map, a, bg, r, stream);
}

// SparseConvTensor.dense() into the split BEV map: hi / lo*2048 fp16 planes [2,B,H,W,D*C] (channel d*C + c).
__global__ void sparse_to_bev_split_kernel(const float4* __restrict__ feat, const int4* __restrict__ coors,
                                           const int* __restrict__ d_rows, int rows_cap, int C4, int D, int H, int W,
                                           size_t plane, __half* __restrict__ bev, int* __restrict__ tile_dist,
                                           int* __restrict__ status) {
    const int rows = min(*d_rows, rows_cap);
    const long long total = (long long)rows * C4;
    tc::F16Range ovf;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i / C4), q = (int)(i % C4);
        const int4 c = __ldg(&coors[r]);
        const float4 v = __ldg(&feat[i]);
        uint32_t h0, h1, l0, l1;
        tc::split_f16x2(v.x, v.y, h0, l0);
        tc::split_f16x2(v.z, v.w, h1, l1);
        ovf.add(l0);
        ovf.add(l1);
        __half* dst = bev + ((((size_t)c.x * H + c.z) * W + c.w) * (size_t)(D * C4) + (size_t)c.y * C4 + q) * 4;
        *(uint2*)dst = make_uint2(h0, h1);
        *(uint2*)(dst + plane) = make_uint2(l0, l1);
        if (tile_dist && q == 0) sassd_mark_conv2d_tiles(tile_dist, c.x, c.z, c.w, H, W);
    }
    tc::report_f16_range(status, ovf.overflowed());
}

extern "C" int sassd_sparse_to_bev_split(const float* feat, const int32_t* coors, const int32_t* d_rows, int rows_cap,
                                         int C, int D, int H, int W, int batch, void* bev_split, int32_t* tile_dist,
                                         sassd_stream_t stream_) {
    return sassd_sparse_to_bev_split_status(feat, coors, d_rows, rows_cap, C, D, H, W, batch, bev_split, tile_dist,
                                            nullptr, stream_);
}

extern "C" int sassd_sparse_to_bev_split_status(const float* feat, const int32_t* coors, const int32_t* d_rows,
                                                int rows_cap, int C, int D, int H, int W, int batch, void* bev_split,
                                                int32_t* tile_dist, int32_t* d_status, sassd_stream_t stream_) {
    if (!feat || !coors || !d_rows || !bev_split || (C & 3) || batch < 1) return SASSD_ERR_ARG;
    if (rows_cap <= 0) return SASSD_OK;
    const size_t plane = (size_t)batch * H * W * D * C;
    sparse_to_bev_split_kernel<<<sassd_grid((long long)rows_cap * (C / 4), 256), 256, 0, (cudaStream_t)stream_>>>(
        (const float4*)feat, (const int4*)coors, d_rows, rows_cap, C / 4, D, H, W, plane, (__half*)bev_split, tile_dist,
        d_status);
    return sassd_check_launch();
}

// Shared helpers for the sassd_b200 CUDA kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/sassd_b200.h"

#define SASSD_EMPTY_KEY (-1)

// Launch-error -> status code (the C ABI never exits or throws; SURVEY.md §5).
static inline int sassd_check_launch() {
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? SASSD_OK : SASSD_ERR_LAUNCH;
}

static inline int sassd_div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// Streaming multiprocessors of the current device (132 on an H100 SXM), queried once per process.
static inline int sassd_num_sms() {
    static const int n = [] {
        int dev = 0, v = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v < 1) {
            cudaGetLastError();
            v = 132;
        }
        return v;
    }();
    return n;
}

// Persistent-style grid sizing: enough CTAs to cover `work` items, capped at
// `ctas_per_sm` resident CTAs per SM (grid-stride loops pick up the rest).
static inline int sassd_grid(long long work, int block, int ctas_per_sm = 8) {
    long long need = (work + block - 1) / block;
    long long cap = (long long)sassd_num_sms() * ctas_per_sm;
    if (need < 1) need = 1;
    return (int)(need < cap ? need : cap);
}

// An active BEV cell (b, y, x) lowers tile_dist of every conv tile within SASSD_TILE_DIST_MAX pixels to its Chebyshev
// distance from the tile rectangle (0 inside the tile).  sassd_conv2d_f16x3_occ compares it with the layer's reach.
__device__ __forceinline__ void sassd_mark_conv2d_tiles(int* __restrict__ tile_dist, int b, int y, int x, int H, int W) {
    const int tiles_y = (H + SASSD_CONV2D_TILE_H - 1) / SASSD_CONV2D_TILE_H;
    const int tiles_x = (W + SASSD_CONV2D_TILE_W - 1) / SASSD_CONV2D_TILE_W;
    const int R = SASSD_TILE_DIST_MAX;
    const int ty0 = max(y - R, 0) / SASSD_CONV2D_TILE_H, ty1 = min(y + R, H - 1) / SASSD_CONV2D_TILE_H;
    const int tx0 = max(x - R, 0) / SASSD_CONV2D_TILE_W, tx1 = min(x + R, W - 1) / SASSD_CONV2D_TILE_W;
    for (int ty = ty0; ty <= ty1; ++ty)
        for (int tx = tx0; tx <= tx1; ++tx) {
            const int y0 = ty * SASSD_CONV2D_TILE_H, x0 = tx * SASSD_CONV2D_TILE_W;
            const int dy = max(max(y0 - y, y - (y0 + SASSD_CONV2D_TILE_H - 1)), 0);
            const int dx = max(max(x0 - x, x - (x0 + SASSD_CONV2D_TILE_W - 1)), 0);
            atomicMin(&tile_dist[(b * tiles_y + ty) * tiles_x + tx], max(dy, dx));
        }
}

// Decoupled look-back for single-pass scans over chunks: a chunk's descriptor is {flag << 32 | value}, flag 0 = not
// published yet, AGG = the chunk's own total, PREFIX = inclusive prefix up to and including the chunk.
#define SASSD_SCAN_AGG 1ull
#define SASSD_SCAN_PREFIX 2ull
// warp-wide look-back over the descriptors of chunks c-1, c-2, ...: returns the exclusive prefix of chunk c
__device__ __forceinline__ int sassd_lookback(volatile unsigned long long* vd, int c, int lane) {
    int base = 0;
    for (int j0 = c - 1; j0 >= 0; j0 -= 32) {
        const int j = j0 - lane;
        unsigned long long d = SASSD_SCAN_PREFIX << 32;            // lanes before chunk 0: an empty prefix
        if (j >= 0) do { d = vd[j]; } while ((d >> 32) == 0ull);
        const unsigned pref = __ballot_sync(0xffffffffu, (d >> 32) == SASSD_SCAN_PREFIX);
        const int first = __ffs(pref) - 1;                     // nearest predecessor with an inclusive prefix
        int v = (pref == 0u || lane <= first) ? (int)(unsigned)d : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        base += v;
        if (pref) break;
    }
    return base;
}

__device__ __forceinline__ uint32_t sassd_hash32(uint32_t k) {
    // Fibonacci hashing followed by a xor-fold; table sizes are powers of two.
    k *= 0x9E3779B1u;
    k ^= k >> 15;
    return k;
}

// Open-addressing insert of a unique key; returns the slot.  keys[] must be
// pre-filled with SASSD_EMPTY_KEY.  `mask` = slots - 1.
__device__ __forceinline__ int sassd_hash_insert_unique(int* __restrict__ keys, uint32_t mask, int key) {
    uint32_t s = sassd_hash32((uint32_t)key) & mask;
    while (true) {
        int prev = atomicCAS(&keys[s], SASSD_EMPTY_KEY, key);
        if (prev == SASSD_EMPTY_KEY || prev == key) return (int)s;
        s = (s + 1) & mask;
    }
}

// Read-only lookup; returns slot or -1.
__device__ __forceinline__ int sassd_hash_find(const int* __restrict__ keys, uint32_t mask, int key) {
    uint32_t s = sassd_hash32((uint32_t)key) & mask;
    while (true) {
        int k = __ldg(&keys[s]);
        if (k == key) return (int)s;
        if (k == SASSD_EMPTY_KEY) return -1;
        s = (s + 1) & mask;
    }
}

// Block-wide exclusive scan of one int per thread (blockDim.x <= 1024, multiple of 32).
// Returns the exclusive prefix; *total receives the block sum.  `smem` needs 33 ints.
__device__ __forceinline__ int sassd_block_exscan(int v, int* smem, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
    int inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += t;
    }
    if (lane == 31) smem[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int w = lane < nwarp ? smem[lane] : 0;
        int winc = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, winc, d);
            if (lane >= d) winc += t;
        }
        smem[lane] = winc - w;           // exclusive warp offsets
        if (lane == 31) smem[32] = winc; // block total
    }
    __syncthreads();
    int res = smem[warp] + inc - v;
    *total = smem[32];
    __syncthreads();
    return res;
}

// Gathered implicit-GEMM convolution on the Hopper tensor cores (wgmma, sm_90a),
// fp32-accurate through a 3-product hi/lo operand split (SASSD_PREC_TF32X3 / SASSD_PREC_F16X3).
//
//   out[m, :] = act( (sum_t  in[row(m,t), :] @ W[t]) * scale + shift )
//
// One persistent CTA per SM, warp-specialised:
//   warps 0-7   consumers : two warpgroups, warpgroup g owns rows 64g..64g+63 of the 128-row tile; they issue
//                           wgmma (M=64, N=NB, K=8 tf32 / 16 f16) from shared memory, lo*hi + hi*lo + hi*hi per
//                           K step into register accumulators, then BN scale/shift, ReLU -> global rows
//   warps 8-15  A producer: two threads per tile row; per (tap, channel chunk) they gather the row's 128 B
//                           (neighbour table / 3x3 window / identity), split every fp32 into hi + lo and store both
//                           into 128B-swizzled K-major shared-memory tiles (generic proxy -> mbarrier; the
//                           consumers fence the proxies before their MMAs read the tiles)
//                           lane 0 of producer warp 8 also issues the cp.async.bulk of the stage's pre-split,
//                           pre-swizzled weight block (16 warps: the register file's four quarters split evenly)
// A work unit is one tile and NB <= 64 of its output channels (two register accumulators of NB/2 floats per thread
// must fit beside the producers' register budget); wider layers walk the tile once per 64-channel part.
//
// Why 3 products: one TF32 pass (10-bit mantissa) cannot hold the 1e-4 parity bar across 22 layers;
// hi = tf32_rn(x), lo = tf32_rn(x - hi), and a*b ~= a_hi*b_hi + a_hi*b_lo + a_lo*b_hi leaves ~2^-21 relative
// error per product (fp16: lo carries a factor 2048, 22 bits survive).
#include <cstdlib>

#include "common.cuh"

#include "tc_common.cuh"

namespace tc {

template <int MODE>
struct RowMapTC {
    const int* nbr;
    int taps, M, H, W;
    __device__ __forceinline__ int operator()(int m, int t, int x, int y) const {
        if (m >= M) return -1;
        if (MODE == SASSD_GCONV_TABLE) return __ldg(&nbr[(size_t)m * taps + t]);
        if (MODE == SASSD_GCONV_ROWS || taps == 1) return m;
        const int dy = t / 3 - 1, dx = t % 3 - 1;
        const int yy = y + dy, xx = x + dx;
        if (yy < 0 || yy >= H || xx < 0 || xx >= W) return -1;
        return m + dy * W + dx;
    }
};

constexpr int GC_PROD_WARPS = 8;
constexpr int GC_THREADS = CONS_THREADS + GC_PROD_WARPS * 32;   // 512
constexpr int GC_WARP_PROD = CONS_THREADS / 32;

template <int NB>
struct Cfg {
    static constexpr int B_TILE_BYTES = NB * 128;                         // per hi / lo
    static constexpr int STAGE_BYTES = 2 * A_TILE_BYTES + 2 * B_TILE_BYTES;
    static constexpr int STAGES = 4;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

// NB = output channels per work unit, bn = padded width of the weight pack (a multiple of NB), nparts = bn / NB
template <int MODE, int NB, int PREC>
__global__ void __launch_bounds__(GC_THREADS, 1)
gconv_tc_kernel(const float* __restrict__ in, const float* __restrict__ wpack, const float* __restrict__ scale,
                const float* __restrict__ shift, const int* __restrict__ nbr, const int* __restrict__ d_rows,
                float* __restrict__ out, int cin, int cout, int taps, int in_stride, int out_stride, int rows_cap,
                int H, int W, int relu, int bn, int nparts, int* __restrict__ status) {
    using C = Cfg<NB>;
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment is required by the 128B swizzle
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_base = base + C::STAGES * C::STAGE_BYTES;
    auto full_a = [&](int s) { return bar_base + 8u * s; };
    auto full_b = [&](int s) { return bar_base + 8u * (C::STAGES + s); };
    auto empty = [&](int s) { return bar_base + 8u * (2 * C::STAGES + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int M = d_rows ? min(__ldg(d_rows), rows_cap) : rows_cap;
    const int nunits = (M + BM - 1) / BM * nparts;
    using PR = Prec<PREC>;
    const int kchunks = (cin + PR::BKC - 1) / PR::BKC;
    const int nchunks = taps * kchunks;

    if (threadIdx.x == 0) {
        for (int s = 0; s < C::STAGES; ++s) {
            mbar_init(full_a(s), GC_PROD_WARPS);   // one elected arrive per producer warp
            mbar_init(full_b(s), 1);
            mbar_init(empty(s), 2);                // one arrive per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp >= GC_WARP_PROD) {
        // ===================== A producers =====================
        const int pt = threadIdx.x - CONS_THREADS;
        const int r = pt & 127;                           // tile row 0..127
        const int hf = pt >> 7;                           // which half of the row's 128-byte chunk this thread fills
        RowMapTC<MODE> rowmap{nbr, taps, M, H, W};
        const uint32_t row_off = (uint32_t)(r >> 3) * 1024u + (uint32_t)(r & 7) * 128u;
        const uint32_t sw = (uint32_t)(r & 7);
        int stage = 0;
        uint32_t phase = 0;
        for (int unit = blockIdx.x; unit < nunits; unit += gridDim.x) {
            const int m = (unit / nparts) * BM + r;
            // pack block of chunk ch: [hi: bn rows][lo: bn rows] of 128 bytes; this unit's NB rows of each
            const uint8_t* wsrc = (const uint8_t*)wpack + (size_t)(unit % nparts) * C::B_TILE_BYTES;
            int x = 0, y = 0;
            if (MODE == SASSD_GCONV_CONV2D) { x = m % W; y = (m / W) % H; }
            // software pipeline: the global loads of the next PF chunks are in flight (register ring) while
            // the current chunk is split, waits for its stage and is stored — the gather is latency-bound
            // (random rows out of L2), so bytes in flight are what buys throughput
            constexpr int NF4H = PR::NF4 / 2;             // float4 loads per thread per chunk
            constexpr int PF = PREC == 0 ? 3 : 2;         // prefetch distance in chunks
            float4 ring[PF][NF4H];
            bool ring_live[PF];                           // false = the slot stands for a missing neighbour (zeros)
            int f_t = 0, f_kc = 0;                        // fetch cursor (tap, channel chunk)
            int f_src = rowmap(m, 0, x, y);
            int f_src_nt = taps > 1 ? rowmap(m, 1, x, y) : -1;   // row index one tap ahead of the cursor
            auto fetch = [&](float4 (&dst)[NF4H], bool& live) {
                const float* rowp = in + (size_t)(f_src < 0 ? 0 : f_src) * in_stride;
                live = f_src >= 0;
#pragma unroll
                for (int c = 0; c < NF4H; ++c) {
                    const int k = f_kc * PR::BKC + (hf * NF4H + c) * 4;
                    dst[c] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (live && k < cin) dst[c] = __ldg((const float4*)(rowp + k));
                }
                if (++f_kc == kchunks) {
                    f_kc = 0;
                    ++f_t;
                    f_src = f_src_nt;
                    f_src_nt = (f_t + 1 < taps) ? rowmap(m, f_t + 1, x, y) : -1;
                }
            };
#pragma unroll
            for (int u = 0; u < PF; ++u)
                if (u < nchunks) fetch(ring[u], ring_live[u]);
            for (int ch0 = 0; ch0 < nchunks; ch0 += PF) {
#pragma unroll
                for (int u = 0; u < PF; ++u) {
                    const int ch = ch0 + u;
                    if (ch >= nchunks) break;
                    float4 (&vn)[NF4H] = ring[u];
                    uint4 ph[4], pl[4];       // this thread's 4 of the 8 16-byte chunks of the hi / lo rows
                    F16Range ovf;             // the lo halves of this chunk (one vote per chunk: no register
                                              // lives across the chunk loop for it)
                    if (!ring_live[u]) {      // missing neighbour (most sparse (row, offset) slots): no split math
#pragma unroll
                        for (int c = 0; c < 4; ++c) { ph[c] = make_uint4(0u, 0u, 0u, 0u); pl[c] = ph[c]; }
                    } else if constexpr (PREC == 0) {
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            float4 hi, lo;
                            split_tf32(vn[c].x, hi.x, lo.x);
                            split_tf32(vn[c].y, hi.y, lo.y);
                            split_tf32(vn[c].z, hi.z, lo.z);
                            split_tf32(vn[c].w, hi.w, lo.w);
                            ph[c] = *reinterpret_cast<const uint4*>(&hi);
                            pl[c] = *reinterpret_cast<const uint4*>(&lo);
                        }
                    } else {
#pragma unroll
                        for (int c = 0; c < 4; ++c) {      // 8 channels (two float4) -> one 16-byte chunk of halfs
                            const float4 a = vn[2 * c], b = vn[2 * c + 1];
                            uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
                            split_f16x2(a.x, a.y, h0, l0);
                            split_f16x2(a.z, a.w, h1, l1);
                            split_f16x2(b.x, b.y, h2, l2);
                            split_f16x2(b.z, b.w, h3, l3);
                            ph[c] = make_uint4(h0, h1, h2, h3);
                            pl[c] = make_uint4(l0, l1, l2, l3);
                            ovf.add(l0); ovf.add(l1); ovf.add(l2); ovf.add(l3);
                        }
                    }
                    report_f16_range(status, ovf.overflowed());
                    if (ch + PF < nchunks) fetch(vn, ring_live[u]);        // refill this ring slot
                    if (lane == 0) {                                        // one polling lane per warp
                        mbar_wait(empty(stage), phase ^ 1u);
                        if (warp == GC_WARP_PROD) {                         // the stage's weight block
                            const uint32_t dst = base + stage * C::STAGE_BYTES + 2 * A_TILE_BYTES;
                            const uint8_t* src = wsrc + (size_t)ch * (2 * bn * 128);
                            mbar_expect_tx(full_b(stage), 2 * C::B_TILE_BYTES);
                            bulk_g2s(dst, src, C::B_TILE_BYTES, full_b(stage));
                            bulk_g2s(dst + C::B_TILE_BYTES, src + (size_t)bn * 128, C::B_TILE_BYTES, full_b(stage));
                        }
                    }
                    __syncwarp();
                    uint8_t* a_hi = smem_raw + (base - smem_u32(smem_raw)) + stage * C::STAGE_BYTES;
                    uint8_t* a_lo = a_hi + A_TILE_BYTES;
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const uint32_t off = row_off + (((uint32_t)(hf * 4 + c) ^ sw) << 4);
                        *(uint4*)(a_hi + off) = ph[c];
                        *(uint4*)(a_lo + off) = pl[c];
                    }
                    // no proxy fence here (it would wait for the prefetch ring's loads still in flight); the
                    // consumers fence after their mbarrier wait
                    __syncwarp();
                    if (lane == 0) mbar_arrive(full_a(stage));
                    if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
                }
            }
        }
    } else {
        // ===================== consumers: MMAs + epilogue =====================
        const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
        // big: hi*hi of the current chunk, added to sum in fp32 RN after every chunk (the tensor core's accumulation
        // truncates: over the 2304-term K of a 3x3 256-channel layer that alone cost 4x the FFMA kernel's error);
        // small: the cross terms of all chunks, 2^-11 smaller
        float big[NB / 2], small[NB / 2], sum[NB / 2];
        int stage = 0;
        uint32_t phase = 0;
        for (int unit = blockIdx.x; unit < nunits; unit += gridDim.x) {
            const int tile = unit / nparts, n0 = (unit % nparts) * NB;
#pragma unroll
            for (int i = 0; i < NB / 2; ++i) { small[i] = 0.f; sum[i] = 0.f; }
            for (int ch = 0; ch < nchunks; ++ch) {
                mbar_wait(full_a(stage), phase);
                fence_proxy_async();        // producers' generic-proxy stores -> visible to the MMAs' async proxy
                mbar_wait(full_b(stage), phase);
                const uint32_t a_hi = base + stage * C::STAGE_BYTES + (uint32_t)wg * (A_TILE_BYTES / 2);
                const uint32_t b_hi = base + stage * C::STAGE_BYTES + 2 * A_TILE_BYTES;
                wgmma_fence();
                mma_chunk_x3<PREC, NB>(big, small, a_hi, a_hi + A_TILE_BYTES, b_hi, b_hi + C::B_TILE_BYTES, true);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs<NB / 2>(big);
                if (t == 0) mbar_arrive(empty(stage));
#pragma unroll
                for (int i = 0; i < NB / 2; ++i) sum[i] = __fadd_rn(sum[i], big[i]);
                if (++stage == C::STAGES) { stage = 0; phase ^= 1u; }
            }
            fence_regs<NB / 2>(small);
            const int r0 = tile * BM + wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);
#pragma unroll
            for (int j = 0; j < NB / 8; ++j) {
                const int n = n0 + 8 * j + 2 * (t & 3);
                float sc[2], sh[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    sc[e] = (scale && n + e < cout) ? __ldg(&scale[n + e]) : 1.f;
                    sh[e] = (shift && n + e < cout) ? __ldg(&shift[n + e]) : 0.f;
                }
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int m = r0 + 8 * i;
                    if (m >= M || n >= cout) continue;
                    float o[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float sm = PREC == 0 ? small[4 * j + 2 * i + e] : small[4 * j + 2 * i + e] * (1.f / kF16LoScale);
                        float val = fmaf(__fadd_rn(sum[4 * j + 2 * i + e], sm), sc[e], sh[e]);
                        if (relu) val = sassd_relu(val);
                        o[e] = val;
                    }
                    float* orow = out + (size_t)m * out_stride;
                    if (n + 1 < cout && (out_stride & 1) == 0) *(float2*)(orow + n) = make_float2(o[0], o[1]);
                    else {
                        orow[n] = o[0];
                        if (n + 1 < cout) orow[n + 1] = o[1];
                    }
                }
            }
        }
    }
}

template <int MODE, int NB, int PREC>
static int launch(const sassd_gconv_desc* d, const float* in, const float* w, const float* scale, const float* shift,
                  const int* nbr, const int* d_rows, float* out, int* status, cudaStream_t stream, int bn) {
    using C = Cfg<NB>;
    auto kern = gconv_tc_kernel<MODE, NB, PREC>;
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES) != cudaSuccess)
            return SASSD_ERR_LAUNCH;
        configured = true;
    }
    const int nparts = bn / NB;
    const int units = sassd_div_up(d->rows_cap, BM) * nparts;
    const int grid = units < sassd_num_sms() ? (units > 0 ? units : 1) : sassd_num_sms();
    kern<<<grid, GC_THREADS, C::SMEM_BYTES, stream>>>(in, w, scale, shift, nbr, d_rows, out, d->cin, d->cout, d->taps,
                                                      d->in_stride, d->out_stride, d->rows_cap, d->H, d->W, d->relu,
                                                      bn, nparts, status);
    return sassd_check_launch();
}

template <int MODE, int PREC>
static int dispatch(const sassd_gconv_desc* d, const float* in, const float* w, const float* scale, const float* shift,
                    const int* nbr, const int* d_rows, float* out, int* st, cudaStream_t s) {
    if (d->cout <= 16) return launch<MODE, 16, PREC>(d, in, w, scale, shift, nbr, d_rows, out, st, s, 16);
    if (d->cout <= 32) return launch<MODE, 32, PREC>(d, in, w, scale, shift, nbr, d_rows, out, st, s, 32);
    if (d->cout <= 64) return launch<MODE, 64, PREC>(d, in, w, scale, shift, nbr, d_rows, out, st, s, 64);
    if (d->cout <= 128) return launch<MODE, 64, PREC>(d, in, w, scale, shift, nbr, d_rows, out, st, s, 128);
    if (d->cout <= 256) return launch<MODE, 64, PREC>(d, in, w, scale, shift, nbr, d_rows, out, st, s, 256);
    return SASSD_ERR_UNSUPPORTED;
}

template <int PREC>
static int dispatch_mode(const sassd_gconv_desc* d, const float* in, const float* w, const float* scale,
                         const float* shift, const int* nbr, const int* d_rows, float* out, int* st, cudaStream_t s) {
    switch (d->mode) {
        case SASSD_GCONV_TABLE: return dispatch<SASSD_GCONV_TABLE, PREC>(d, in, w, scale, shift, nbr, d_rows, out, st, s);
        case SASSD_GCONV_CONV2D: return dispatch<SASSD_GCONV_CONV2D, PREC>(d, in, w, scale, shift, nbr, d_rows, out, st, s);
        case SASSD_GCONV_ROWS: return dispatch<SASSD_GCONV_ROWS, PREC>(d, in, w, scale, shift, nbr, d_rows, out, st, s);
    }
    return SASSD_ERR_ARG;
}

}  // namespace tc

// `weight` for these paths is the pre-split, pre-swizzled pack produced by sassd_gconv_pack:
//   TF32X3: [taps*ceil(cin/32)][hi|lo][BN rows (n)][32 fp32]   F16X3: [taps*ceil(cin/64)][hi|lo][BN][64 fp16]
// every row is 128 bytes, its 16-byte chunks XOR-swizzled by (n & 7).
int sassd_gconv_tc(const sassd_gconv_desc* d, const float* in, const float* weight, const float* scale,
                   const float* shift, const int32_t* nbr, const int32_t* d_rows, float* out, int32_t* d_status,
                   cudaStream_t stream) {
    if (d->precision == SASSD_PREC_TF32X3)
        return tc::dispatch_mode<0>(d, in, weight, scale, shift, nbr, d_rows, out, d_status, stream);
    if (d->precision == SASSD_PREC_F16X3)
        return tc::dispatch_mode<1>(d, in, weight, scale, shift, nbr, d_rows, out, d_status, stream);
    return SASSD_ERR_ARG;
}

static inline int tc_bn(int cout) { return cout <= 16 ? 16 : cout <= 32 ? 32 : cout <= 64 ? 64 : cout <= 128 ? 128 : 256; }

// Weight packer (device): W [taps, cin, cout] fp32 -> the layouts above.  One thread per packed element.
template <int PREC>
__global__ void pack_kernel(const float* __restrict__ w, int taps, int cin, int cout, int bn, void* __restrict__ out_) {
    constexpr int BKC = tc::Prec<PREC>::BKC;
    constexpr int EPC = PREC == 0 ? 4 : 8;                // elements per 16-byte chunk
    const int kchunks = (cin + BKC - 1) / BKC;
    const long long per_chunk = 2LL * bn * BKC;
    const long long total = (long long)taps * kchunks * per_chunk;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long ch = i / per_chunk;
        long long rem = i % per_chunk;
        const int part = (int)(rem / (bn * BKC));         // 0 = hi, 1 = lo
        rem %= (bn * BKC);
        const int n = (int)(rem / BKC);
        const int pos = (int)(rem % BKC);                 // physical element slot inside the 128-byte row
        const int chunk16 = pos / EPC, e = pos % EPC;
        const int kk = ((chunk16 ^ (n & 7)) * EPC) + e;   // logical k stored at this physical slot
        const int t = (int)(ch / kchunks), kc = (int)(ch % kchunks);
        const int k = kc * BKC + kk;
        float v = 0.f;
        if (k < cin && n < cout) v = w[((size_t)t * cin + k) * cout + n];
        if constexpr (PREC == 0) {
            float hi, lo;
            tc::split_tf32(v, hi, lo);
            ((float*)out_)[i] = part == 0 ? hi : lo;
        } else {
            float hi, lo;
            tc::split_f16(v, hi, lo);
            ((__half*)out_)[i] = __float2half_rn(part == 0 ? hi : lo);
        }
    }
}

extern "C" size_t sassd_gconv_pack_bytes(int taps, int cin, int cout, int precision) {
    const int bn = tc_bn(cout);
    if (precision == SASSD_PREC_TF32X3) return (size_t)taps * ((cin + 31) / 32) * 2 * bn * 128;
    if (precision == SASSD_PREC_F16X3) return (size_t)taps * ((cin + 63) / 64) * 2 * bn * 128;
    return 0;
}

extern "C" int sassd_gconv_pack(const float* weight, int taps, int cin, int cout, int precision, void* packed,
                                sassd_stream_t stream_) {
    if (!weight || !packed || taps <= 0 || cin <= 0 || cout <= 0 || cout > 256) return SASSD_ERR_ARG;
    const int bn = tc_bn(cout);
    if (precision == SASSD_PREC_TF32X3) {
        const long long total = (long long)taps * ((cin + 31) / 32) * 2 * bn * 32;
        pack_kernel<0><<<sassd_grid(total, 256), 256, 0, (cudaStream_t)stream_>>>(weight, taps, cin, cout, bn, packed);
    } else if (precision == SASSD_PREC_F16X3) {
        const long long total = (long long)taps * ((cin + 63) / 64) * 2 * bn * 64;
        pack_kernel<1><<<sassd_grid(total, 256), 256, 0, (cudaStream_t)stream_>>>(weight, taps, cin, cout, bn, packed);
    } else {
        return SASSD_ERR_ARG;
    }
    return sassd_check_launch();
}

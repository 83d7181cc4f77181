// Gathered implicit-GEMM convolution, CUDA-core FFMA path (SASSD_PREC_FP32).
//
//   out[m, :] = act( (sum_t  in[row(m,t), :] @ W[t]) * scale + shift )
//
// One kernel family serves the 13 ruled sparse convs + the 1x1x1 conv of VxNet
// (spconv indice_conv semantics, cmn.py:192-231), the 8 BEVNet convs
// (cmn.py:264-282), the three SSDRotateHead 1x1 convs (ssd_rotate_head.py:218-231)
// and the two PSWarpHead convs (:424-429).  Output-stationary: a CTA owns
// BM=128 output rows x BN output channels, loops over the taps, gathers the
// input rows named by the neighbour table (or computed for dense 3x3 windows),
// and writes every output row exactly once — no atomics, deterministic, BN+ReLU
// fused in the epilogue.  Taps with no neighbour in the whole tile are skipped.
//
// Algorithmic bytes per rule pair (SURVEY.md §8d): 4*Cin + 4*Cout + 8.
#include "common.cuh"

#define GC_BM 128
#define GC_THREADS 256

template <int MODE>
struct RowMap {
    const int* nbr;
    int taps, M, H, W;
    __device__ __forceinline__ int operator()(int m, int t) const {
        if (m >= M) return -1;
        if (MODE == SASSD_GCONV_TABLE) return __ldg(&nbr[(size_t)m * taps + t]);
        if (MODE == SASSD_GCONV_ROWS) return m;
        // CONV2D: m = (b*H + y)*W + x, tap t = ky*3 + kx (taps == 9) or the centre (taps == 1)
        if (taps == 1) return m;
        const int x = m % W, y = (m / W) % H;
        const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
        if (yy < 0 || yy >= H || xx < 0 || xx >= W) return -1;
        return m + (t / 3 - 1) * W + (t % 3 - 1);
    }
};

template <int MODE, int BN, int BK>
__global__ void __launch_bounds__(GC_THREADS, 2)
gconv_ffma_kernel(const float* __restrict__ in, const float* __restrict__ weight, const float* __restrict__ scale,
                  const float* __restrict__ shift, const int* __restrict__ nbr, const int* __restrict__ d_rows,
                  float* __restrict__ out, int cin, int cout, int taps, int in_stride, int out_stride, int rows_cap,
                  int H, int W, int relu) {
    constexpr int TN = BN / 16;                 // output channels per thread
    constexpr int A_F4 = GC_BM * BK / 4;        // float4 loads per A tile
    constexpr int A_PER_T = (A_F4 + GC_THREADS - 1) / GC_THREADS;
    constexpr int B_F4 = BK * BN / 4;
    constexpr int B_PER_T = (B_F4 + GC_THREADS - 1) / GC_THREADS;
    constexpr int QK = BK / 4;                  // float4 per A row slice

    __shared__ __align__(16) float As[2][BK][GC_BM + 4];
    __shared__ __align__(16) float Bs[2][BK][BN];

    const int M = d_rows ? min(__ldg(d_rows), rows_cap) : rows_cap;
    const int n0 = blockIdx.y * BN;
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    RowMap<MODE> rowmap{nbr, taps, M, H, W};
    const int ntiles = (M + GC_BM - 1) / GC_BM;
    // persistent over row tiles: the grid is sized from the capacity, the loop from the device-side row count
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int m0 = tile * GC_BM;

    float acc[8][TN];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    // per-thread A-load assignment: element e -> (row = e / QK, q = e % QK)
    int a_row[A_PER_T], a_q[A_PER_T], a_idx[A_PER_T];
#pragma unroll
    for (int j = 0; j < A_PER_T; ++j) {
        const int e = tid + j * GC_THREADS;
        a_row[j] = e / QK;
        a_q[j] = e % QK;
        a_idx[j] = -1;
    }
    float4 a_reg[A_PER_T], b_reg[B_PER_T];

    int t = -1, kc = cin;  // position of the slice held in the prefetch registers
    bool have = false;

    // advance (t, kc) to the next slice with at least one valid row; fetch it into registers
    auto prefetch = [&]() {
        kc += BK;
        if (kc >= cin) {
            kc = 0;
            while (true) {
                ++t;
                if (t >= taps) { have = false; return; }
                int any = 0;
#pragma unroll
                for (int j = 0; j < A_PER_T; ++j) {
                    a_idx[j] = (tid + j * GC_THREADS < A_F4) ? rowmap(m0 + a_row[j], t) : -1;
                    any |= (a_idx[j] >= 0);
                }
                if (__syncthreads_or(any)) break;
            }
        }
        have = true;
#pragma unroll
        for (int j = 0; j < A_PER_T; ++j) {
            a_reg[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (a_idx[j] >= 0)
                a_reg[j] = __ldg((const float4*)(in + (size_t)a_idx[j] * in_stride + kc + a_q[j] * 4));
        }
        const float* wt = weight + ((size_t)t * cin + kc) * cout;
#pragma unroll
        for (int j = 0; j < B_PER_T; ++j) {
            const int e = tid + j * GC_THREADS;
            b_reg[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (e < B_F4) {
                const int kk = e / (BN / 4), nq = e % (BN / 4);
                const int n = n0 + nq * 4;
                const float* p = wt + (size_t)kk * cout + n;
                if (n + 3 < cout && (cout & 3) == 0) b_reg[j] = __ldg((const float4*)p);
                else {
                    if (n + 0 < cout) b_reg[j].x = __ldg(p + 0);
                    if (n + 1 < cout) b_reg[j].y = __ldg(p + 1);
                    if (n + 2 < cout) b_reg[j].z = __ldg(p + 2);
                    if (n + 3 < cout) b_reg[j].w = __ldg(p + 3);
                }
            }
        }
    };

    prefetch();
    int buf = 0;
    while (have) {
        // registers -> shared (A transposed to k-major)
#pragma unroll
        for (int j = 0; j < A_PER_T; ++j) {
            if (tid + j * GC_THREADS < A_F4) {
                const int r = a_row[j], k4 = a_q[j] * 4;
                As[buf][k4 + 0][r] = a_reg[j].x;
                As[buf][k4 + 1][r] = a_reg[j].y;
                As[buf][k4 + 2][r] = a_reg[j].z;
                As[buf][k4 + 3][r] = a_reg[j].w;
            }
        }
#pragma unroll
        for (int j = 0; j < B_PER_T; ++j) {
            const int e = tid + j * GC_THREADS;
            if (e < B_F4) *(float4*)&Bs[buf][e / (BN / 4)][(e % (BN / 4)) * 4] = b_reg[j];
        }
        __syncthreads();
        prefetch();  // global loads of the next slice overlap the FFMA block below
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float a[8], b[TN];
            *(float4*)&a[0] = *(const float4*)&As[buf][kk][ty * 8];
            *(float4*)&a[4] = *(const float4*)&As[buf][kk][ty * 8 + 4];
            if (TN >= 4) {
#pragma unroll
                for (int j = 0; j < TN; j += 4) *(float4*)&b[j] = *(const float4*)&Bs[buf][kk][tx * TN + j];
            } else {
#pragma unroll
                for (int j = 0; j < TN; ++j) b[j] = Bs[buf][kk][tx * TN + j];
            }
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        buf ^= 1;
        // the next iteration writes the other buffer; the __syncthreads() after that write orders it
        // against this iteration's reads of `buf^1` two iterations later.
    }

    // epilogue: folded BatchNorm / bias, ReLU, one coalesced store per row
    float sc[TN], sh[TN];
#pragma unroll
    for (int j = 0; j < TN; ++j) {
        const int n = n0 + tx * TN + j;
        sc[j] = (n < cout && scale) ? __ldg(&scale[n]) : 1.f;
        sh[j] = (n < cout && shift) ? __ldg(&shift[n]) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + ty * 8 + i;
        if (m >= M) continue;
        float* po = out + (size_t)m * out_stride + n0 + tx * TN;
        float v[TN];
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            v[j] = fmaf(acc[i][j], sc[j], sh[j]);
            if (relu) v[j] = fmaxf(v[j], 0.f);
        }
        if (TN >= 4 && (out_stride & 3) == 0 && n0 + tx * TN + TN <= cout) {
#pragma unroll
            for (int j = 0; j < TN; j += 4) *(float4*)(po + j) = *(const float4*)&v[j];
        } else {
#pragma unroll
            for (int j = 0; j < TN; ++j)
                if (n0 + tx * TN + j < cout) po[j] = v[j];
        }
    }
    __syncthreads();  // smem tiles are reused by the next row tile
    }  // tile loop
}

template <int MODE, int BN, int BK>
static int launch_ffma(const sassd_gconv_desc* d, const float* in, const float* w, const float* scale,
                       const float* shift, const int* nbr, const int* d_rows, float* out, cudaStream_t stream) {
    int gx = sassd_div_up(d->rows_cap, GC_BM);
    if (gx > sassd_num_sms() * 4) gx = sassd_num_sms() * 4;
    dim3 grid(gx, sassd_div_up(d->cout, BN));
    gconv_ffma_kernel<MODE, BN, BK><<<grid, GC_THREADS, 0, stream>>>(in, w, scale, shift, nbr, d_rows, out, d->cin,
                                                                     d->cout, d->taps, d->in_stride, d->out_stride,
                                                                     d->rows_cap, d->H, d->W, d->relu);
    return sassd_check_launch();
}

template <int MODE>
static int dispatch_ffma(const sassd_gconv_desc* d, const float* in, const float* w, const float* scale,
                         const float* shift, const int* nbr, const int* d_rows, float* out, cudaStream_t s) {
    const bool k4 = (d->cin % 16) != 0;  // Cin = 4 (first sparse layer) or other multiples of 4
    if (d->cout <= 16) return k4 ? launch_ffma<MODE, 16, 4>(d, in, w, scale, shift, nbr, d_rows, out, s)
                                 : launch_ffma<MODE, 16, 16>(d, in, w, scale, shift, nbr, d_rows, out, s);
    if (d->cout <= 32) return k4 ? launch_ffma<MODE, 32, 4>(d, in, w, scale, shift, nbr, d_rows, out, s)
                                 : launch_ffma<MODE, 32, 16>(d, in, w, scale, shift, nbr, d_rows, out, s);
    if (d->cout <= 64) return k4 ? launch_ffma<MODE, 64, 4>(d, in, w, scale, shift, nbr, d_rows, out, s)
                                 : launch_ffma<MODE, 64, 16>(d, in, w, scale, shift, nbr, d_rows, out, s);
    return k4 ? launch_ffma<MODE, 128, 4>(d, in, w, scale, shift, nbr, d_rows, out, s)
              : launch_ffma<MODE, 128, 16>(d, in, w, scale, shift, nbr, d_rows, out, s);
}

int sassd_gconv_tc(const sassd_gconv_desc* d, const float* in, const float* weight, const float* scale,
                   const float* shift, const int32_t* nbr, const int32_t* d_rows, float* out, cudaStream_t stream);

extern "C" int sassd_gconv(const sassd_gconv_desc* d, const float* in, const float* weight, const float* scale,
                           const float* shift, const int32_t* nbr, const int32_t* d_rows, float* out,
                           sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!d || !in || !weight || !out) return SASSD_ERR_ARG;
    if (d->cin <= 0 || (d->cin & 3) || d->cout <= 0 || d->taps <= 0 || (d->in_stride & 3) || d->rows_cap < 0)
        return SASSD_ERR_ARG;
    if (d->mode == SASSD_GCONV_TABLE && !nbr) return SASSD_ERR_ARG;
    if (d->mode == SASSD_GCONV_CONV2D && !(d->taps == 9 || d->taps == 1)) return SASSD_ERR_ARG;
    if (d->mode == SASSD_GCONV_ROWS && d->taps != 1) return SASSD_ERR_ARG;
    if (d->rows_cap == 0) return SASSD_OK;
    if (d->precision == SASSD_PREC_TF32X3 || d->precision == SASSD_PREC_F16X3)
        return sassd_gconv_tc(d, in, weight, scale, shift, nbr, d_rows, out, stream);
    if (d->precision != SASSD_PREC_FP32) return SASSD_ERR_ARG;
    switch (d->mode) {
        case SASSD_GCONV_TABLE: return dispatch_ffma<SASSD_GCONV_TABLE>(d, in, weight, scale, shift, nbr, d_rows, out, stream);
        case SASSD_GCONV_CONV2D: return dispatch_ffma<SASSD_GCONV_CONV2D>(d, in, weight, scale, shift, nbr, d_rows, out, stream);
        case SASSD_GCONV_ROWS: return dispatch_ffma<SASSD_GCONV_ROWS>(d, in, weight, scale, shift, nbr, d_rows, out, stream);
    }
    return SASSD_ERR_ARG;
}

// ---------------------------------------------------------------------------
// dense(): scatter the last sparse layer's rows into the (pre-zeroed) NHWC BEV map
// ---------------------------------------------------------------------------
__global__ void sparse_to_bev_kernel(const float4* __restrict__ feat, const int4* __restrict__ coors,
                                     const int* __restrict__ d_rows, int rows_cap, int C4, int D, int H, int W,
                                     float4* __restrict__ bev) {
    const int rows = min(*d_rows, rows_cap);
    const long long total = (long long)rows * C4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i / C4), q = (int)(i % C4);
        const int4 c = __ldg(&coors[r]);  // (b, d, y, x)
        bev[(((size_t)c.x * H + c.z) * W + c.w) * (size_t)(D * C4) + (size_t)c.y * C4 + q] = __ldg(&feat[i]);
    }
}

extern "C" int sassd_sparse_to_bev(const float* feat, const int32_t* coors, const int32_t* d_rows, int rows_cap, int C,
                                   int D, int H, int W, float* bev, sassd_stream_t stream_) {
    if (!feat || !coors || !d_rows || !bev || (C & 3)) return SASSD_ERR_ARG;
    if (rows_cap <= 0) return SASSD_OK;
    sparse_to_bev_kernel<<<sassd_grid((long long)rows_cap * (C / 4), 256), 256, 0, (cudaStream_t)stream_>>>(
        (const float4*)feat, (const int4*)coors, d_rows, rows_cap, C / 4, D, H, W, (float4*)bev);
    return sassd_check_launch();
}

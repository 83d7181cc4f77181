// Head tail: second_box_decode + get_guided_anchors, PSWarp sampling.
// (mmdet/models/single_stage_heads/ssd_rotate_head.py:53-91,307-372,374-414,431-447)
//
// The reference loops over the batch in Python with ~15 tiny kernels and two
// nonzero() syncs per frame; here the whole batch is two launches (count, emit)
// with an order-preserving compaction, counts stay on the device.
#include "common.cuh"

#define DS_CHUNK 1024  // anchors per CTA (256 threads x 4 consecutive anchors)

struct HeadLayout {
    int H, W, ncls, stride;   // stride = floats per pixel of the NHWC head map
    int cls_off, dir_off;     // channel offsets of conv_cls / conv_dir_cls (conv_box at 0)
    int n_anchors;
};

__device__ __forceinline__ float sigmoidf_(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

// anchor a = ((cls_a*H + y)*W + x)*2 + rot
__device__ __forceinline__ void anchor_decompose(const HeadLayout& L, int a, int& cls_a, int& pix, int& rot) {
    rot = a & 1;
    const int t = a >> 1;
    const int hw = L.H * L.W;
    cls_a = t / hw;
    pix = t - cls_a * hw;
}

// max_c sigmoid(cls logits) and its argmax like torch.max on CPU: the first maximum on ties, and the first NaN wins
// both the value and the index (so a NaN class score is never selected: NaN > thr is false)
__device__ __forceinline__ float anchor_score(const HeadLayout& L, const float* __restrict__ head_b, int a, int& label) {
    int cls_a, pix, rot;
    anchor_decompose(L, a, cls_a, pix, rot);
    const float* p = head_b + (size_t)pix * L.stride + L.cls_off + cls_a * (2 * L.ncls) + rot * L.ncls;
    float best = sigmoidf_(__ldg(p));
    label = 0;
    for (int c = 1; c < L.ncls; ++c) {
        const float s = sigmoidf_(__ldg(p + c));
        if (s > best || (s != s && best == best)) { best = s; label = c; }
    }
    return best;
}

__global__ void __launch_bounds__(256)
ds_count_kernel(const float* __restrict__ head, HeadLayout L, const uint8_t* __restrict__ mask, float thr,
                int nchunks, int* __restrict__ chunk_count) {
    __shared__ int s_red[8];
    const int b = blockIdx.y, chunk = blockIdx.x;
    const float* head_b = head + (size_t)b * L.H * L.W * L.stride;
    const uint8_t* mask_b = mask + (size_t)b * L.n_anchors;
    int cnt = 0;
    const int a0 = chunk * DS_CHUNK + threadIdx.x * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int a = a0 + j;
        if (a < L.n_anchors && mask_b[a]) {
            int lb;
            cnt += anchor_score(L, head_b, a, lb) > thr ? 1 : 0;
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, d);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int i = 0; i < 8; ++i) t += s_red[i];
        chunk_count[b * nchunks + chunk] = t;
    }
}

__global__ void __launch_bounds__(256)
ds_emit_kernel(const float* __restrict__ head, HeadLayout L, const float* __restrict__ anchors,
               size_t anchor_frame_stride, const uint8_t* __restrict__ mask, float thr, int nchunks, const int* __restrict__ chunk_count,
               float* __restrict__ boxes, int* __restrict__ labels, int* __restrict__ index, int* __restrict__ d_k,
               int k_cap, int* __restrict__ status) {
    __shared__ int s_scan[33];
    __shared__ int s_base;
    const int b = blockIdx.y, chunk = blockIdx.x;
    // exclusive offset of this chunk = sum of the earlier chunks' counts
    int part = 0;
    for (int c = threadIdx.x; c < chunk; c += 256) part += chunk_count[b * nchunks + c];
    int tot;
    sassd_block_exscan(part, s_scan, &tot);
    if (threadIdx.x == 0) s_base = tot;
    __syncthreads();
    const int base = s_base;

    const float* head_b = head + (size_t)b * L.H * L.W * L.stride;
    const uint8_t* mask_b = mask + (size_t)b * L.n_anchors;
    const int a0 = chunk * DS_CHUNK + threadIdx.x * 4;
    int flags = 0, lbl[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int a = a0 + j;
        lbl[j] = 0;
        if (a < L.n_anchors && mask_b[a] && anchor_score(L, head_b, a, lbl[j]) > thr) flags |= 1 << j;
    }
    int total;
    int pos = base + sassd_block_exscan(__popc(flags), s_scan, &total);
    if (chunk == nchunks - 1 && threadIdx.x == 0) {
        int k = base + total;
        if (k > k_cap) { atomicOr(status, SASSD_FLAG_GUIDED_CAP); k = k_cap; }
        d_k[b] = k;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (!(flags & (1 << j))) continue;
        if (pos < k_cap) {
            const int a = a0 + j;
            int cls_a, pix, rot;
            anchor_decompose(L, a, cls_a, pix, rot);
            const float* px = head_b + (size_t)pix * L.stride;
            const float* e = px + cls_a * 14 + rot * 7;               // xt yt zt wt lt ht rt
            const float* an = anchors + (size_t)b * anchor_frame_stride + (size_t)a * 7;   // xa ya za wa la ha ra
            const float xa = __ldg(an + 0), ya = __ldg(an + 1), za = __ldg(an + 2), wa = __ldg(an + 3),
                        la = __ldg(an + 4), ha = __ldg(an + 5), ra = __ldg(an + 6);
            // second_box_decode, op by op in fp32 without contraction (torch evaluates each op separately)
            const float zac = __fadd_rn(za, __fdiv_rn(ha, 2.f));
            const float diag = sqrtf(__fadd_rn(__fmul_rn(la, la), __fmul_rn(wa, wa)));
            const float xg = __fadd_rn(__fmul_rn(__ldg(e + 0), diag), xa);
            const float yg = __fadd_rn(__fmul_rn(__ldg(e + 1), diag), ya);
            float zg = __fadd_rn(__fmul_rn(__ldg(e + 2), ha), zac);
            const float wg = __fmul_rn(expf(__ldg(e + 3)), wa);
            const float lg = __fmul_rn(expf(__ldg(e + 4)), la);
            const float hg = __fmul_rn(expf(__ldg(e + 5)), ha);
            float rg = __fadd_rn(__ldg(e + 6), ra);
            zg = __fsub_rn(zg, __fdiv_rn(hg, 2.f));
            // direction classifier: dir_label = torch.max's argmax (first max on ties, the first NaN wins); flip when
            // (r > 0) != dir_label
            const float* dp = px + L.dir_off + cls_a * 4 + rot * 2;
            const float d0 = __ldg(dp + 0), d1 = __ldg(dp + 1);
            const bool dir_label = d0 == d0 && (d1 > d0 || d1 != d1);
            if ((rg > 0.f) != dir_label) rg = __fadd_rn(rg, 3.14159274101257324f);
            float* ob = boxes + ((size_t)b * k_cap + pos) * 7;
            ob[0] = xg; ob[1] = yg; ob[2] = zg; ob[3] = wg; ob[4] = lg; ob[5] = hg; ob[6] = rg;
            labels[(size_t)b * k_cap + pos] = lbl[j];
            index[(size_t)b * k_cap + pos] = a;
        }
        ++pos;
    }
}

extern "C" size_t sassd_decode_select_workspace_bytes(int batch, int n_anchors) {
    return (size_t)batch * ((n_anchors + DS_CHUNK - 1) / DS_CHUNK) * sizeof(int);
}

extern "C" int sassd_decode_select(const float* head, int head_stride, int batch, int H, int W, int num_class,
                                   const float* anchors, int anchors_per_frame, const uint8_t* mask, int n_anchors,
                                   float thr, float* boxes,
                                   int32_t* labels, int32_t* index, int32_t* d_k, int k_cap, int32_t* d_status,
                                   void* ws, size_t ws_bytes, sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!head || !anchors || !mask || !boxes || !labels || !index || !d_k || !d_status || !ws) return SASSD_ERR_ARG;
    if (batch < 1 || num_class < 1 || n_anchors != num_class * H * W * 2 || k_cap < 1) return SASSD_ERR_ARG;
    const int na = 2 * num_class;
    if (head_stride < na * 7 + na * num_class + na * 2) return SASSD_ERR_ARG;
    if (ws_bytes < sassd_decode_select_workspace_bytes(batch, n_anchors)) return SASSD_ERR_WORKSPACE;
    HeadLayout L;
    L.H = H; L.W = W; L.ncls = num_class; L.stride = head_stride;
    L.cls_off = na * 7; L.dir_off = na * 7 + na * num_class; L.n_anchors = n_anchors;
    const int nchunks = (n_anchors + DS_CHUNK - 1) / DS_CHUNK;
    dim3 grid(nchunks, batch);
    ds_count_kernel<<<grid, 256, 0, stream>>>(head, L, mask, thr, nchunks, (int*)ws);
    ds_emit_kernel<<<grid, 256, 0, stream>>>(head, L, anchors, anchors_per_frame ? (size_t)n_anchors * 7 : 0, mask, thr, nchunks, (const int*)ws, boxes, labels, index,
                                             d_k, k_cap, d_status);
    return sassd_check_launch();
}

// ---------------------------------------------------------------------------
// PSWarp: one warp per guided box, lane p < 28 = part p = i*7 + j of the 4x7 window.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
pswarp_kernel(const float* __restrict__ feat, int stride, int H, int W, const float* __restrict__ boxes,
              const int* __restrict__ d_k, int k_cap, float off_x, float off_y, float sscale,
              float* __restrict__ scores) {
    // torch.linspace(-.5, .5, 4) and (-.5, .5, 7) in fp32, bit patterns as torch produces them
    const float lin4[4] = {-0.5f, __int_as_float(0xBE2AAAAA), __int_as_float(0x3E2AAAAA), 0.5f};
    const float lin7[7] = {-0.5f, __int_as_float(0xBEAAAAAA), __int_as_float(0xBE2AAAAA), __int_as_float(0xB2800000),
                           __int_as_float(0x3E2AAAAA), __int_as_float(0x3EAAAAAA), 0.5f};
    const int b = blockIdx.y;
    const int k = min(d_k[b], k_cap);
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    const float* feat_b = feat + (size_t)b * H * W * stride;
    for (int i = blockIdx.x * wpb + (threadIdx.x >> 5); i < k; i += gridDim.x * wpb) {
        const float* bx = boxes + ((size_t)b * k_cap + i) * 7;
        const float xg = __ldg(bx + 0), yg = __ldg(bx + 1), wg = __ldg(bx + 3), lg = __ldg(bx + 4), rg = __ldg(bx + 6);
        float val = 0.f;
        if (lane < 28) {
            const int pi = lane / 7, pj = lane % 7;
            const float c = cosf(rg), s = sinf(rg);
            const float xx = __fmul_rn(lin4[pi], wg), yy = __fmul_rn(lin7[pj], lg);
            // gen_sample_grid (:393-397)
            float x = __fadd_rn(__fadd_rn(__fmul_rn(xx, c), __fmul_rn(yy, s)), xg);
            float y = __fadd_rn(__fsub_rn(__fmul_rn(yy, c), __fmul_rn(xx, s)), yg);
            x = __fmul_rn(__fadd_rn(x, off_x), sscale);
            y = __fmul_rn(__fadd_rn(y, off_y), sscale);
            // normalisation (:410-412) then grid_sample's align_corners=True un-normalisation
            float gx = __fsub_rn(__fmul_rn(__fdiv_rn(x, (float)(W - 1)), 2.f), 1.f);
            float gy = __fsub_rn(__fmul_rn(__fdiv_rn(y, (float)(H - 1)), 2.f), 1.f);
            const float ix = __fmul_rn(__fdiv_rn(__fadd_rn(gx, 1.f), 2.f), (float)(W - 1));
            const float iy = __fmul_rn(__fdiv_rn(__fadd_rn(gy, 1.f), 2.f), (float)(H - 1));
            const float fx = floorf(ix), fy = floorf(iy);
            const float w_e = __fsub_rn(ix, fx), w_w = __fsub_rn(1.f, w_e);
            const float w_s = __fsub_rn(iy, fy), w_n = __fsub_rn(1.f, w_s);
            // Each tap's validity is decided on the floats (false for NaN), and only a valid tap's corner is converted
            // to int: converting an out-of-range float is undefined, and an int x0 + 1 may wrap (x0 = INT_MAX gave
            // x1 = INT_MIN, which passed x1 >= 0 once the compiler rewrote it as x0 > -2).  Off the map a tap adds
            // exactly 0, however far off it is.
            const bool vx0 = fx >= 0.f && fx < (float)W, vx1 = fx >= -1.f && fx < (float)(W - 1);
            const bool vy0 = fy >= 0.f && fy < (float)H, vy1 = fy >= -1.f && fy < (float)(H - 1);
            const int x0 = vx0 || vx1 ? (int)fx : 0, y0 = vy0 || vy1 ? (int)fy : 0, x1 = x0 + 1, y1 = y0 + 1;
            const float* fp = feat_b + lane;
            float acc = 0.f;
            if (vy0 && vx0) acc = __fadd_rn(acc, __fmul_rn(__ldg(fp + ((size_t)y0 * W + x0) * stride), __fmul_rn(w_n, w_w)));
            if (vy0 && vx1) acc = __fadd_rn(acc, __fmul_rn(__ldg(fp + ((size_t)y0 * W + x1) * stride), __fmul_rn(w_n, w_e)));
            if (vy1 && vx0) acc = __fadd_rn(acc, __fmul_rn(__ldg(fp + ((size_t)y1 * W + x0) * stride), __fmul_rn(w_s, w_w)));
            if (vy1 && vx1) acc = __fadd_rn(acc, __fmul_rn(__ldg(fp + ((size_t)y1 * W + x1) * stride), __fmul_rn(w_s, w_e)));
            // A non-finite sample coordinate (a box with an infinite or NaN centre, size or yaw) has no position on
            // the map: the part is NaN, so the box's score is NaN and the rescoring threshold drops it.  The float
            // predicates above alone would give it 0, a finite score.
            val = isfinite(ix) && isfinite(iy) ? acc : __int_as_float(0x7fc00000);
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) val += __shfl_down_sync(0xffffffffu, val, d);
        if (lane == 0) scores[(size_t)b * k_cap + i] = __fdiv_rn(val, 28.f);
    }
}

extern "C" int sassd_pswarp(const float* feat, int feat_stride, int batch, int H, int W, const float* boxes,
                            const int32_t* d_k, int k_cap, float off_x, float off_y, float spatial_scale,
                            float* scores, sassd_stream_t stream_) {
    if (!feat || !boxes || !d_k || !scores || feat_stride < 28 || batch < 1 || k_cap < 1) return SASSD_ERR_ARG;
    const int wpb = 8;
    int gx = (k_cap + wpb - 1) / wpb;
    if (gx > sassd_num_sms() * 4) gx = sassd_num_sms() * 4;
    dim3 grid(gx, batch);
    pswarp_kernel<<<grid, wpb * 32, 0, (cudaStream_t)stream_>>>(feat, feat_stride, H, W, boxes, d_k, k_cap, off_x,
                                                                off_y, spatial_scale, scores);
    return sassd_check_launch();
}

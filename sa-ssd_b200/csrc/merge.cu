// Detections of several single-class models, merged per frame (detectors.DetectorSet): member m's det
// [batch,cap_m,9] / d_ndet [batch] blocks, as sassd_rescore_nms writes them, gathered into one [batch,sum cap_m,9]
// block.  Frame f's rows are member 0's first d_ndet_0[f] rows, then member 1's, and so on, each row copied bit for bit
// except its label (column 8), which gains the member's offset into the set's class list.  No NMS across members: the
// merged rows are the concatenation a user would build from the members' result files.
//
// One CTA per frame: thread 0 reads the members' counts and their running offsets into shared memory, then the block
// copies every member's rows with a stride loop over floats.  No host synchronisation and no status flag:
// graph-capturable.  The member descriptors travel in the kernel's parameter block.
#include "common.cuh"

#define MD_THREADS 256

struct MergeMembers {
    const float* det[SASSD_MERGE_MAX];
    const int32_t* ndet[SASSD_MERGE_MAX];
    int cap[SASSD_MERGE_MAX];
    float label_offset[SASSD_MERGE_MAX];
};

__global__ void __launch_bounds__(MD_THREADS)
merge_detections_kernel(const MergeMembers mm, int n_members, int cap_out, float* __restrict__ det_out,
                        int32_t* __restrict__ d_ndet_out) {
    __shared__ int s_n[SASSD_MERGE_MAX], s_base[SASSD_MERGE_MAX];
    const int f = blockIdx.x;
    if (threadIdx.x == 0) {
        int base = 0;
        for (int m = 0; m < n_members; ++m) {
            const int n = min(max(mm.ndet[m][f], 0), mm.cap[m]);
            s_n[m] = n;
            s_base[m] = base;
            base += n;
        }
        d_ndet_out[f] = base;
    }
    __syncthreads();
    float* out = det_out + (size_t)f * cap_out * 9;
    for (int m = 0; m < n_members; ++m) {
        const float* src = mm.det[m] + (size_t)f * mm.cap[m] * 9;
        float* dst = out + (size_t)s_base[m] * 9;
        const int nv = s_n[m] * 9;
        const float off = mm.label_offset[m];
        for (int i = threadIdx.x; i < nv; i += MD_THREADS) {
            const float v = src[i];
            dst[i] = (i % 9 == 8) ? __fadd_rn(v, off) : v;
        }
    }
}

extern "C" int sassd_merge_detections(const float* const* host_dets, const int32_t* const* host_ndets,
                                      const int* host_caps, const int* host_label_offsets, int n_members, int batch,
                                      float* det, int32_t* d_ndet, sassd_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!host_dets || !host_ndets || !host_caps || !host_label_offsets || !det || !d_ndet) return SASSD_ERR_ARG;
    if (n_members < 1 || n_members > SASSD_MERGE_MAX || batch < 1) return SASSD_ERR_ARG;
    MergeMembers mm = {};
    long long cap_out = 0;
    for (int m = 0; m < n_members; ++m) {
        if (!host_dets[m] || !host_ndets[m] || host_caps[m] < 1 || host_label_offsets[m] < 0) return SASSD_ERR_ARG;
        mm.det[m] = host_dets[m];
        mm.ndet[m] = host_ndets[m];
        mm.cap[m] = host_caps[m];
        mm.label_offset[m] = (float)host_label_offsets[m];
        cap_out += host_caps[m];
    }
    if (cap_out > (1 << 24)) return SASSD_ERR_ARG;
    merge_detections_kernel<<<batch, MD_THREADS, 0, stream>>>(mm, n_members, (int)cap_out, det, d_ndet);
    return sassd_check_launch();
}

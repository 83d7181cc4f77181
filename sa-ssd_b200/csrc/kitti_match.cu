// The KITTI evaluator's cleaning and matching on the device (mmdet/core/evaluation/kitti_eval.py:39-92 clean_data,
// :95-154 box / 3-D overlaps, :17-36 get_thresholds, :164-283 compute_statistics_jit, :295-342
// fused_compute_statistics), for K detection sets against one ground truth and any number of min-overlap rows at once:
//
//   sassd_kitti_eval_flags     ignore flags of every GT and detection row for every (class, difficulty);
//   sassd_kitti_eval_overlaps  the 2-D box, BEV and 3-D overlap matrices of every (set, frame), from the rotated
//                              overlaps of sassd_rotate_overlap_eval;
//   sassd_kitti_eval_match     for every job (set, class, difficulty, metric, min-overlap row): the true-positive
//                              scores, the 41 sampled score thresholds and the per-threshold (tp, fp, fn, similarity)
//                              sums over all frames, i.e. the host matcher's `pr` array.
//
// Every fp64 expression is written with round-to-nearest intrinsics in numpy's (or the host matcher's) operation order
// and without FMA contraction, so that each array equals what the host path (kitti_eval.py + sassd_kitti_match)
// computes bit for bit.  The one transcendental, cos() of the AOS similarity, comes from a host table
// (sassd_kitti_aos_table) made with the host matcher's libm, since the device cos() rounds differently.
#include <cmath>
#include <cstdint>

#include "common.cuh"

namespace {

constexpr int kThresh = 41;                  // sampled recall positions (get_thresholds' num_sample_pts)
constexpr int kMatchCtas = 1024, kMatchThreads = 256;   // persistent grid of the two matching passes
constexpr long long kScratchThreads = (long long)kMatchCtas * kMatchThreads;
constexpr double kNo = -10000000.0;          // compute_statistics_jit's NO_DETECTION

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// The reference's min(a, b) and max(a, b) (numba / Python: the second argument when it compares below / above the
// first, else the first), in place of fmin / fmax, which drop a NaN from either side: a NaN coordinate then gives the
// reference's overlap, NaN or a number, whichever side it is on.  In the DontCare test the order cannot change the
// outcome (a NaN detection coordinate makes the quotient's denominator, the detection's area, NaN), but it is kept
// the reference's there too, so that every min / max of the evaluation reads the same.
__device__ __forceinline__ double ref_min(double a, double b) { return b < a ? b : a; }
__device__ __forceinline__ double ref_max(double a, double b) { return b > a ? b : a; }

// ------------------------------------------------------------------------------------------------------ flags
// The ground distance of a camera-frame row (x, y, z, ...): sqrt(x * x + z * z), numpy's operation order.
__device__ __forceinline__ double ground_range(const double* cam) {
    return __dsqrt_rn(dadd(dmul(cam[0], cam[0]), dmul(cam[2], cam[2])));
}

// Whether range r falls in difficulty entry d's bin [ranges[2d], ranges[2d+1]).  No ranges, or an entry whose lower
// edge is -inf, means no range test (every row, a NaN range included); otherwise a NaN range falls in no bin.
__device__ __forceinline__ bool in_bin(const double* ranges, int d, double r) {
    if (!ranges) return true;
    const double lo = ranges[2 * d], hi = ranges[2 * d + 1];
    return lo == -INFINITY || (lo <= r && r < hi);
}

// clean_data (kitti_eval.py:39-92) for every row: GT flags 0 evaluate / 1 ignore / -1 other class, detection flags
// 1 too low / 0 the class / -1 other class.  limits[3 * d + (0, 1, 2)] = (max occlusion, max truncation, min height)
// of difficulty entry d; classes[2 * c] is class c's name id, classes[2 * c + 1] the id of the name that counts as
// "don't care" for it (van for car, person_sitting for pedestrian) or -1.  With ranges, a GT row of the class outside
// entry d's bin is ignored (1) as a GT harder than the difficulty is, and a detection of the class outside it is
// ignored (1) as a low one is; gt_range / dt_range (when given) receive every row's ground distance.
__global__ void eval_flags_kernel(int ngt, const int32_t* __restrict__ gt_name, const double* __restrict__ gt_occ,
                                  const double* __restrict__ gt_trunc, const double* __restrict__ gt_bbox,
                                  const double* __restrict__ gt_cam, int ndt, const int32_t* __restrict__ dt_name,
                                  const double* __restrict__ dt_bbox, const double* __restrict__ dt_cam, int nclass,
                                  const int32_t* __restrict__ classes, int ndiff, const double* __restrict__ limits,
                                  const double* __restrict__ ranges, int8_t* __restrict__ ign_gt,
                                  int8_t* __restrict__ ign_dt, int32_t* __restrict__ n_valid,
                                  double* __restrict__ gt_range, double* __restrict__ dt_range) {
    const long long rows = (long long)ngt + ndt, total = rows * nclass * ndiff;
    for (long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x; w < total; w += (long long)gridDim.x * blockDim.x) {
        const int cd = (int)(w / rows), c = cd / ndiff, d = cd % ndiff;
        const long long r = w % rows;
        const int cls = classes[2 * c], alt = classes[2 * c + 1];
        const double max_occ = limits[3 * d], max_trunc = limits[3 * d + 1], min_h = limits[3 * d + 2];
        if (r < ngt) {
            const double rg = (ranges || gt_range) ? ground_range(gt_cam + 7 * r) : 0.0;
            if (cd == 0 && gt_range) gt_range[r] = rg;
            const int nm = gt_name[r];
            const int valid = nm == cls ? 1 : (alt >= 0 && nm == alt ? 0 : -1);
            const double h = dsub(gt_bbox[4 * r + 3], gt_bbox[4 * r + 1]);
            const bool ignore = gt_occ[r] > max_occ || gt_trunc[r] > max_trunc || h <= min_h || !in_bin(ranges, d, rg);
            const int f = (valid == 1 && !ignore) ? 0 : ((valid == 0 || (ignore && valid == 1)) ? 1 : -1);
            ign_gt[(long long)cd * ngt + r] = (int8_t)f;
            if (f == 0) atomicAdd(&n_valid[cd], 1);
        } else {
            const long long j = r - ngt;
            const double rd = (ranges || dt_range) ? ground_range(dt_cam + 7 * j) : 0.0;
            if (cd == 0 && dt_range) dt_range[j] = rd;
            const double h = fabs(dsub(dt_bbox[4 * j + 3], dt_bbox[4 * j + 1]));
            ign_dt[(long long)cd * ndt + j] =
                (int8_t)(h < min_h ? 1 : (dt_name[j] == cls ? (in_bin(ranges, d, rd) ? 0 : 1) : -1));
        }
    }
}

// --------------------------------------------------------------------------------------------------- overlaps
// Block b = k * nframes + f is set k's frame f: detections [dt_off[b], dt_off[b+1]) against GT rows
// [gt_off[f], gt_off[f+1]), every matrix row-major [detection, GT] at ov_off[b].  cam rows are (x, y, z, l, h, w, ry).
__global__ void eval_overlaps_kernel(int nsets, int nframes, const int32_t* __restrict__ gt_off,
                                     const int32_t* __restrict__ dt_off, const long long* __restrict__ ov_off,
                                     const double* __restrict__ gt_cam, const double* __restrict__ dt_cam,
                                     const double* __restrict__ gt_bbox, const double* __restrict__ dt_bbox,
                                     const float* __restrict__ bev_iou, const float* __restrict__ bev_inter,
                                     double* __restrict__ ov_bbox, double* __restrict__ ov_bev, double* __restrict__ ov_3d) {
    for (int b = blockIdx.y; b < nsets * nframes; b += gridDim.y) {
        const int f = b % nframes;
        const int g0 = gt_off[f], ng = gt_off[f + 1] - g0, d0 = dt_off[b], nd = dt_off[b + 1] - d0;
        const long long total = (long long)ng * nd, o0 = ov_off[b];
        for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total;
             p += (long long)gridDim.x * blockDim.x) {
            const int j = (int)(p / ng), i = (int)(p % ng);
            // image_box_overlap(dt, gt, criterion=-1) (kitti_eval.py:95-122, vectorised in kitti_eval.py)
            const double* b4 = dt_bbox + 4 * (long long)(d0 + j);
            const double* q4 = gt_bbox + 4 * (long long)(g0 + i);
            const double iw = dsub(ref_min(b4[2], q4[2]), ref_max(b4[0], q4[0]));
            const double ih = dsub(ref_min(b4[3], q4[3]), ref_max(b4[1], q4[1]));
            double v = 0.0;
            if (iw > 0 && ih > 0) {
                const double area_b = dmul(dsub(b4[2], b4[0]), dsub(b4[3], b4[1]));
                const double area_q = dmul(dsub(q4[2], q4[0]), dsub(q4[3], q4[1]));
                const double inter = dmul(iw, ih);
                v = ddiv(inter, dsub(dadd(area_b, area_q), inter));
            }
            ov_bbox[o0 + p] = v;
            ov_bev[o0 + p] = (double)bev_iou[o0 + p];
            // _d3_from_bev (kitti_eval.py:130-154): the height overlap times the float32 BEV intersection area, the
            // quotient rounded to float32
            const double* bc = dt_cam + 7 * (long long)(d0 + j);
            const double* qc = gt_cam + 7 * (long long)(g0 + i);
            const float rinc = bev_inter[o0 + p];
            const double hw = dsub(ref_min(bc[1], qc[1]), ref_max(dsub(bc[1], bc[4]), dsub(qc[1], qc[4])));
            // a BEV intersection that is not > 0 (0 or NaN) is kept, as d3_box_overlap_kernel leaves it
            double v3 = rinc > 0.f ? 0.0 : (double)rinc;
            if (rinc > 0.f && hw > 0) {
                const double inc = dmul(hw, (double)rinc);
                const double a1 = dmul(dmul(bc[3], bc[4]), bc[5]), a2 = dmul(dmul(qc[3], qc[4]), qc[5]);
                v3 = (double)(float)ddiv(inc, dsub(dadd(a1, a2), inc));
            }
            ov_3d[o0 + p] = v3;
        }
    }
}

// ---------------------------------------------------------------------------------------------------- matching
struct Job {
    int k, c, d, m, o;
};

__device__ __forceinline__ Job decode_job(const SassdKittiEvalDesc& e, long long job) {
    Job j;
    j.o = (int)(job % e.nover); job /= e.nover;
    j.m = (int)(job % 3); job /= 3;
    j.d = (int)(job % e.ndiff); job /= e.ndiff;
    j.c = (int)(job % e.nclass);
    j.k = (int)(job / e.nclass);
    return j;
}

// One frame of one job, everything the matching reads.
struct Frame {
    const double* ov;        // [nd, ng]
    const double* aos;       // [nd, ng] (1 + cos(gt alpha - dt alpha)) / 2, or null
    const int8_t *igt, *idt;
    const int32_t* dc;       // DontCare flag of each GT row
    const double *score, *dt_bbox, *gt_bbox;
    int ng, nd;
};

__device__ __forceinline__ Frame frame_of(const SassdKittiEvalDesc& e, const Job& jb, int f) {
    Frame fr;
    const int b = jb.k * e.nframes + f, g0 = e.gt_off[f], d0 = e.dt_off[b];
    const long long ngt = e.gt_off[e.nframes], ndt = e.dt_off[e.nsets * e.nframes];
    const long long cd = (long long)jb.c * e.ndiff + jb.d;
    fr.ng = e.gt_off[f + 1] - g0;
    fr.nd = e.dt_off[b + 1] - d0;
    const double* ovs[3] = {e.ov_bbox, e.ov_bev, e.ov_3d};
    fr.ov = ovs[jb.m] + e.ov_off[b];
    fr.aos = (jb.m == 0 && e.aos_table && e.compute_aos[jb.k]) ? e.aos_table + e.ov_off[b] : nullptr;
    fr.igt = e.ign_gt + cd * ngt + g0;
    fr.idt = e.ign_dt + cd * ndt + d0;
    fr.dc = e.gt_dc + g0;
    fr.score = e.dt_score + d0;
    fr.dt_bbox = e.dt_bbox + 4 * (long long)d0;
    fr.gt_bbox = e.gt_bbox + 4 * (long long)g0;
    return fr;
}

__device__ __forceinline__ double min_overlap_of(const SassdKittiEvalDesc& e, const Job& jb) {
    return e.min_overlaps[((long long)jb.o * 3 + jb.m) * e.nclass + jb.c];   // [nover, metric, class]
}

// Pass 1 (compute_fp=False): append the score of every true positive to its job's score region.  One thread per
// (job, frame); `asg` is this thread's assigned-detection scratch, stride kScratchThreads.
// With `frames`, each score's frame goes to the same slot of it.
__global__ void __launch_bounds__(kMatchThreads) eval_tp_scores_kernel(SassdKittiEvalDesc e, long long njobs,
                                                                     char* __restrict__ asg_ws,
                                                                     double* __restrict__ scores,
                                                                     int32_t* __restrict__ n_scores,
                                                                     int32_t* __restrict__ frames = nullptr) {
    const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    char* asg = asg_ws + tid;
    for (long long w = tid; w < njobs * e.nframes; w += kScratchThreads) {
        const long long job = w / e.nframes;
        const Job jb = decode_job(e, job);
        const Frame fr = frame_of(e, jb, (int)(w % e.nframes));
        if (fr.ng == 0 || fr.nd == 0) continue;
        const double min_ov = min_overlap_of(e, jb);
        const long long base = e.score_off[job], cap = e.score_off[job + 1] - base;
        for (int j = 0; j < fr.nd; ++j) asg[j * kScratchThreads] = 0;
        for (int i = 0; i < fr.ng; ++i) {
            const int gi = fr.igt[i];
            if (gi == -1) continue;
            int det = -1;
            double valid = kNo;
            for (int j = 0; j < fr.nd; ++j) {
                if (fr.idt[j] == -1 || asg[j * kScratchThreads]) continue;
                if (fr.ov[(long long)j * fr.ng + i] > min_ov && fr.score[j] > valid) {
                    det = j;
                    valid = fr.score[j];
                }
            }
            if (valid == kNo) continue;      // a missed GT (fn) is not counted in this pass
            if (gi == 1 || fr.idt[det] == 1) {
                asg[det * kScratchThreads] = 1;
            } else {
                const int slot = atomicAdd(&n_scores[job], 1);
                if (slot < cap) {
                    scores[base + slot] = fr.score[det];
                    if (frames) frames[base + slot] = (int32_t)(w % e.nframes);
                }
                asg[det * kScratchThreads] = 1;
            }
        }
    }
}

// Sort the first n of a job's P (a power of two) scores descending, bitonic over the whole region padded with -inf,
// by the whole CTA; `tag` (or null) is permuted with them.
__device__ void sort_desc(double* s, int32_t* tag, long long n, long long P) {
    for (long long i = n + threadIdx.x; i < P; i += blockDim.x) {
        s[i] = -INFINITY;
        if (tag) tag[i] = -1;
    }
    __syncthreads();
    for (long long k = 2; k <= P; k <<= 1)
        for (long long jj = k >> 1; jj > 0; jj >>= 1) {
            for (long long i = threadIdx.x; i < P; i += blockDim.x) {
                const long long l = i ^ jj;
                if (l > i) {
                    const double a = s[i], b = s[l];
                    if ((i & k) == 0 ? a < b : a > b) {      // descending runs where (i & k) == 0
                        s[i] = b;
                        s[l] = a;
                        if (tag) {
                            const int32_t t = tag[i];
                            tag[i] = tag[l];
                            tag[l] = t;
                        }
                    }
                }
            }
            __syncthreads();
        }
}

// get_thresholds (kitti_eval.py:17-36): sort each job's scores descending (bitonic, in its power-of-two region), then
// pick the scores at the 41 sampled recall positions.  One CTA per job.
__global__ void eval_thresholds_kernel(SassdKittiEvalDesc e, double* __restrict__ scores,
                                       const int32_t* __restrict__ n_scores, double* __restrict__ thresholds,
                                       int32_t* __restrict__ n_thresh) {
    const long long job = blockIdx.x;
    const Job jb = decode_job(e, job);
    double* s = scores + e.score_off[job];
    const long long P = e.score_off[job + 1] - e.score_off[job];
    const long long n = n_scores[job] < P ? n_scores[job] : P;
    sort_desc(s, nullptr, n, P);
    if (threadIdx.x != 0) return;
    const double num_gt = (double)e.n_valid[(long long)jb.c * e.ndiff + jb.d];
    const double step = 1.0 / (kThresh - 1.0);
    double cur = 0.0;
    int nt = 0;
    for (long long i = 0; i < n && nt < kThresh; ++i) {
        const double l_recall = ddiv((double)(i + 1), num_gt);
        const double r_recall = i < n - 1 ? ddiv((double)(i + 2), num_gt) : l_recall;
        if (dsub(r_recall, cur) < dsub(cur, l_recall) && i < n - 1) continue;
        thresholds[job * kThresh + nt++] = s[i];
        cur = dadd(cur, step);
    }
    n_thresh[job] = nt;
}

// np.sum of [0] * nz followed by vals[0 .. n - nz) (stride kScratchThreads): numpy's pairwise summation (blocks of 8
// partial sums up to 128 elements, halves rounded down to a multiple of 8 above), as the host matcher restates it.
// The recursion runs on an explicit stack of pending left halves.
__device__ double pairwise_leaf(const double* vals, int nz, int lo, int n) {
    auto at = [&](int e) { return lo + e < nz ? 0.0 : vals[(long long)(lo + e - nz) * kScratchThreads]; };
    if (n < 8) {
        double s = 0.0;
        for (int i = 0; i < n; ++i) s = dadd(s, at(i));
        return s;
    }
    double r[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = at(k);
    int i = 8;
    for (; i + 8 <= n; i += 8)
#pragma unroll
        for (int k = 0; k < 8; ++k) r[k] = dadd(r[k], at(i + k));
    double s = dadd(dadd(dadd(r[0], r[1]), dadd(r[2], r[3])), dadd(dadd(r[4], r[5]), dadd(r[6], r[7])));
    for (; i < n; ++i) s = dadd(s, at(i));
    return s;
}

__device__ double pairwise_sum(const double* vals, int nz, int n) {
    int lo_s[32], n_s[32];
    double left_s[32];
    bool right_s[32];
    int depth = 0, lo = 0;
    for (;;) {
        while (n > 128) {                          // descend into left halves
            int n2 = n / 2;
            n2 -= n2 % 8;
            lo_s[depth] = lo; n_s[depth] = n; right_s[depth] = false;
            ++depth;
            n = n2;
        }
        double r = pairwise_leaf(vals, nz, lo, n);
        for (;;) {                                 // climb until a split still owes its right half
            if (depth == 0) return r;
            const int d = depth - 1;
            int n2 = n_s[d] / 2;
            n2 -= n2 % 8;
            if (!right_s[d]) {
                left_s[d] = r; right_s[d] = true;
                lo = lo_s[d] + n2; n = n_s[d] - n2;
                break;
            }
            r = dadd(left_s[d], r);
            depth = d;
        }
    }
}

// Where frame_statistics records its assignment (the match table): per GT row the matched detection (its row in the
// set, or -1) and their overlap (0 when unmatched); per detection row its SASSD_KITTI_DT_* state.
struct Record {
    int32_t* gt_det;
    double* gt_ov;
    int8_t* dt_state;
    int row0;            // the set's row of the frame's first detection
};

// compute_statistics_jit with compute_fp=True (kitti_eval.py:164-283) for one frame at one threshold; with kRecord
// also the frame's assignment into `rec`.
template <bool kRecord>
__device__ void frame_statistics(const Frame& fr, int metric, double min_ov, double thresh, char* asg, double* vals,
                                 int* tp_out, int* fp_out, int* fn_out, double* sim_out, const Record& rec = Record{}) {
    const long long S = kScratchThreads;
    int tp = 0, fp = 0, fn = 0, nv = 0;
    for (int j = 0; j < fr.nd; ++j) asg[j * S] = 0;
    if constexpr (kRecord) {
        for (int i = 0; i < fr.ng; ++i) { rec.gt_det[i] = -1; rec.gt_ov[i] = 0.0; }
        for (int j = 0; j < fr.nd; ++j) rec.dt_state[j] = SASSD_KITTI_DT_NOT_COUNTED;
    }
    for (int i = 0; i < fr.ng; ++i) {
        const int gi = fr.igt[i];
        if (gi == -1) continue;
        int det = -1;
        double valid = kNo, max_ov = 0.0;
        bool assigned_ign = false;
        for (int j = 0; j < fr.nd; ++j) {
            const int dj = fr.idt[j];
            if (dj == -1 || asg[j * S] || fr.score[j] < thresh) continue;
            const double ov = fr.ov[(long long)j * fr.ng + i];
            if (ov > min_ov && (ov > max_ov || assigned_ign) && dj == 0) {
                max_ov = ov; det = j; valid = 1; assigned_ign = false;
            } else if (ov > min_ov && valid == kNo && dj == 1) {
                det = j; valid = 1; assigned_ign = true;
            }
        }
        if (valid == kNo && gi == 0) {
            ++fn;
        } else if (valid != kNo && (gi == 1 || fr.idt[det] == 1)) {
            asg[det * S] = 1;
            if constexpr (kRecord) rec.dt_state[det] = SASSD_KITTI_DT_IGNORED;
        } else if (valid != kNo) {
            ++tp;
            if (fr.aos) vals[(long long)nv++ * S] = fr.aos[(long long)det * fr.ng + i];
            asg[det * S] = 1;
            if constexpr (kRecord) rec.dt_state[det] = SASSD_KITTI_DT_TP;
        }
        if constexpr (kRecord)
            if (valid != kNo) {
                rec.gt_det[i] = rec.row0 + det;
                rec.gt_ov[i] = fr.ov[(long long)det * fr.ng + i];
            }
    }
    for (int j = 0; j < fr.nd; ++j)
        if (!(asg[j * S] || fr.idt[j] == -1 || fr.idt[j] == 1 || fr.score[j] < thresh)) {
            ++fp;
            if constexpr (kRecord) rec.dt_state[j] = SASSD_KITTI_DT_FP;
        }
    int nstuff = 0;
    if (metric == 0)
        for (int i = 0; i < fr.ng; ++i) {
            if (!fr.dc[i]) continue;
            const double* q = fr.gt_bbox + 4 * i;       // a DontCare box
            for (int j = 0; j < fr.nd; ++j) {
                if (asg[j * S] || fr.idt[j] == -1 || fr.idt[j] == 1 || fr.score[j] < thresh) continue;
                const double* b = fr.dt_bbox + 4 * j;    // image_box_overlap with criterion 0
                const double iw = dsub(ref_min(b[2], q[2]), ref_max(b[0], q[0]));
                if (iw <= 0) continue;
                const double ih = dsub(ref_min(b[3], q[3]), ref_max(b[1], q[1]));
                if (ih <= 0) continue;
                if (ddiv(dmul(iw, ih), dmul(dsub(b[2], b[0]), dsub(b[3], b[1]))) > min_ov) {
                    asg[j * S] = 1;
                    ++nstuff;
                    if constexpr (kRecord) rec.dt_state[j] = SASSD_KITTI_DT_DONTCARE;
                }
            }
        }
    fp -= nstuff;
    double sim = 0.0;
    if (fr.aos) sim = (tp > 0 || fp > 0) ? pairwise_sum(vals, fp > 0 ? fp : 0, (fp > 0 ? fp : 0) + nv) : -1.0;
    *tp_out = tp; *fp_out = fp; *fn_out = fn; *sim_out = sim;
}

// Pass 2 (fused_compute_statistics): one CTA per (job, threshold), its threads over the frames.  The counts are summed
// in any order; the similarity is summed in frame order, as the host accumulates pr[t, 3].
__global__ void __launch_bounds__(kMatchThreads) eval_pr_kernel(SassdKittiEvalDesc e, long long njobs,
                                                              char* __restrict__ asg_ws, double* __restrict__ vals_ws,
                                                              const double* __restrict__ thresholds,
                                                              const int32_t* __restrict__ n_thresh,
                                                              double* __restrict__ pr) {
    __shared__ double s_sim[kMatchThreads];
    __shared__ unsigned long long s_cnt[3];
    const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    char* asg = asg_ws + tid;
    double* vals = vals_ws + tid;
    for (long long w = blockIdx.x; w < njobs * kThresh; w += gridDim.x) {
        const long long job = w / kThresh;
        const int t = (int)(w % kThresh);
        if (t >= n_thresh[job]) continue;                  // uniform over the CTA
        const Job jb = decode_job(e, job);
        const double min_ov = min_overlap_of(e, jb), thresh = thresholds[w];
        const bool aos = jb.m == 0 && e.aos_table && e.compute_aos[jb.k];
        if (threadIdx.x < 3) s_cnt[threadIdx.x] = 0;
        long long tp = 0, fp = 0, fn = 0;
        double sim_sum = 0.0;
        for (int f0 = 0; f0 < e.nframes; f0 += blockDim.x) {
            const int f = f0 + threadIdx.x;
            double sim = -1.0;
            if (f < e.nframes) {
                int a, b, c;
                frame_statistics<false>(frame_of(e, jb, f), jb.m, min_ov, thresh, asg, vals, &a, &b, &c, &sim);
                tp += a; fp += b; fn += c;
            }
            if (aos) {
                s_sim[threadIdx.x] = sim;
                __syncthreads();
                if (threadIdx.x == 0) {
                    const int nf = min((int)blockDim.x, e.nframes - f0);
                    for (int i = 0; i < nf; ++i)
                        if (s_sim[i] != -1.0) sim_sum = dadd(sim_sum, s_sim[i]);
                }
                __syncthreads();
            }
        }
        __syncthreads();
        atomicAdd(&s_cnt[0], (unsigned long long)tp);
        atomicAdd(&s_cnt[1], (unsigned long long)fp);
        atomicAdd(&s_cnt[2], (unsigned long long)fn);
        __syncthreads();
        if (threadIdx.x == 0) {
            double* o = pr + 4 * w;
            o[0] = (double)(long long)s_cnt[0];
            o[1] = (double)(long long)s_cnt[1];
            o[2] = (double)(long long)s_cnt[2];
            o[3] = sim_sum;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------- match table
constexpr double kPi = 3.141592653589793, kTwoPi = 6.283185307179586;

// The TP errors of a 3-D-metric true positive, GT row g against detection row q (camera rows x, y, z, l, h, w, ry):
// ATE the BEV centre distance, ASE 1 - IoU of the boxes aligned at one centre and heading, AOE the heading difference
// wrapped to [0, pi].  fp64 in a fixed order with sqrt the only non-arithmetic operation, as kitti_eval.tp_errors.
__device__ void tp_errors(const double* g, const double* q, double* out) {
    const double dx = dsub(q[0], g[0]), dz = dsub(q[2], g[2]);
    out[0] = __dsqrt_rn(dadd(dmul(dx, dx), dmul(dz, dz)));
    const double vi = dmul(dmul(fmin(q[3], g[3]), fmin(q[4], g[4])), fmin(q[5], g[5]));
    const double vg = dmul(dmul(g[3], g[4]), g[5]), vd = dmul(dmul(q[3], q[4]), q[5]);
    out[1] = dsub(1.0, ddiv(vi, dsub(dadd(vg, vd), vi)));
    const double d = dsub(q[6], g[6]);
    out[2] = fmin(fabs(dsub(d, dmul(kTwoPi, floor(ddiv(dadd(d, kPi), kTwoPi))))), kPi);
}

// compute_statistics_jit's assignment (compute_fp=True, a threshold below every score) of every (set, class,
// difficulty entry < ndiff, metric) job at min-overlap row `row`, one thread per (job, frame), written out instead of
// summed; each 3-D-metric job also writes its TP errors (NaN for a GT row without a true positive).
__global__ void __launch_bounds__(kMatchThreads) eval_assign_kernel(SassdKittiEvalDesc e, int row, int ndiff,
                                                                  long long njobs, char* __restrict__ asg_ws,
                                                                  const double* __restrict__ gt_cam,
                                                                  const double* __restrict__ dt_cam,
                                                                  int32_t* __restrict__ gt_det,
                                                                  double* __restrict__ gt_ov,
                                                                  int8_t* __restrict__ dt_state,
                                                                  double* __restrict__ tp_err) {
    const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    char* asg = asg_ws + tid;
    const long long ngt = e.gt_off[e.nframes], ndt = e.dt_off[e.nsets * e.nframes];
    for (long long w = tid; w < njobs * e.nframes; w += kScratchThreads) {
        const long long job = w / e.nframes;             // ((k * nclass + c) * ndiff + d) * 3 + m
        const int f = (int)(w % e.nframes);
        Job jb;
        jb.m = (int)(job % 3);
        jb.d = (int)(job / 3 % ndiff);
        jb.c = (int)(job / 3 / ndiff % e.nclass);
        jb.k = (int)(job / 3 / ndiff / e.nclass);
        jb.o = row;
        Frame fr = frame_of(e, jb, f);
        fr.aos = nullptr;                                // the table sums no AOS similarity: no `vals` scratch
        const int b = jb.k * e.nframes + f, g0 = e.gt_off[f], d0 = e.dt_off[b];
        const long long cdm = ((long long)jb.c * ndiff + jb.d) * 3 + jb.m;
        Record rec;
        rec.gt_det = gt_det + job * ngt + g0;
        rec.gt_ov = gt_ov + job * ngt + g0;
        rec.dt_state = dt_state + cdm * ndt + d0;
        rec.row0 = d0 - e.dt_off[jb.k * e.nframes];
        int tp, fp, fn;
        double sim;
        frame_statistics<true>(fr, jb.m, min_overlap_of(e, jb), -INFINITY, asg, nullptr, &tp, &fp, &fn, &sim, rec);
        if (jb.m != 2) continue;
        double* err = tp_err + ((((long long)jb.k * e.nclass + jb.c) * ndiff + jb.d) * ngt + g0) * 3;
        for (int i = 0; i < fr.ng; ++i) {
            const int j = rec.gt_det[i] - rec.row0;
            if (j >= 0 && rec.dt_state[j] == SASSD_KITTI_DT_TP) {
                tp_errors(gt_cam + 7 * (long long)(g0 + i), dt_cam + 7 * (long long)(d0 + j), err + 3 * i);
            } else {
                err[3 * i] = err[3 * i + 1] = err[3 * i + 2] = __longlong_as_double(0x7ff8000000000000LL);
            }
        }
    }
}


// --------------------------------------------------------------------------------------------------- bootstrap
// A bootstrap replicate is a list of the split's frames drawn with replacement.  Its matching needs no new overlaps:
// pass 2 reads the threshold only through `score < thresh`, so a frame's (tp, fp, fn, similarity) at threshold t is its
// state at the smallest of its own scores >= t, or the state with every scored detection inactive when there is none
// (a NaN score is active at every threshold).  Each (job, frame) keeps that step table once; a replicate's per-threshold
// sums are then lookups over its list.

// The first table entry of (job, frame f): the job's block of tab_off, then set k's frames, nd + 1 entries each.
__device__ __forceinline__ long long step_base(const SassdKittiEvalDesc& e, const Job& jb, long long job,
                                               const int64_t* tab_off, int f) {
    const int b0 = jb.k * e.nframes;
    return tab_off[job] + (e.dt_off[b0 + f] - e.dt_off[b0]) + f;
}

// One thread per (job, frame): entry 0 is the state with every scored detection inactive (frame_statistics at +inf),
// entries 1..m the states at the frame's distinct non-NaN scores of detections the job does not skip (flag != -1), in
// descending score order; tab_n[job * nframes + f] = m.
__global__ void __launch_bounds__(kMatchThreads) boot_steps_kernel(SassdKittiEvalDesc e, long long njobs,
                                                                 char* __restrict__ asg_ws,
                                                                 double* __restrict__ vals_ws,
                                                                 const int64_t* __restrict__ tab_off,
                                                                 double* __restrict__ tab_score,
                                                                 int32_t* __restrict__ tab_cnt,
                                                                 double* __restrict__ tab_sim,
                                                                 int32_t* __restrict__ tab_n) {
    const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    char* asg = asg_ws + tid;
    double* vals = vals_ws + tid;
    for (long long w = tid; w < njobs * e.nframes; w += kScratchThreads) {
        const long long job = w / e.nframes;
        const int f = (int)(w % e.nframes);
        const Job jb = decode_job(e, job);
        const Frame fr = frame_of(e, jb, f);
        const double min_ov = min_overlap_of(e, jb);
        const long long base = step_base(e, jb, job, tab_off, f);
        double thresh = INFINITY;
        int m = 0;
        for (;;) {
            int tp, fp, fn;
            double sim;
            frame_statistics<false>(fr, jb.m, min_ov, thresh, asg, vals, &tp, &fp, &fn, &sim);
            tab_score[base + m] = thresh;
            tab_cnt[3 * (base + m)] = tp;
            tab_cnt[3 * (base + m) + 1] = fp;
            tab_cnt[3 * (base + m) + 2] = fn;
            tab_sim[base + m] = sim;
            // the next distinct score down: the largest below the last one (any, +inf included, the first time)
            bool found = false;
            double next = 0.0;
            for (int j = 0; j < fr.nd; ++j) {
                const double sc = fr.score[j];
                if (fr.idt[j] == -1 || sc != sc || (m > 0 && !(sc < thresh))) continue;
                if (!found || sc > next) { next = sc; found = true; }
            }
            if (!found) break;
            thresh = next;
            ++m;
        }
        tab_n[w] = m;
    }
}

// get_thresholds over replicate r's true positives: job's sorted scores, entry i counted weight[r, frame of i] times
// (copies of one score are interchangeable), at recall positions over the replicate's valid GT count num_gt[r, cd].
// One thread per (job, replicate), replicates fastest.
__global__ void boot_thresholds_kernel(SassdKittiEvalDesc e, long long njobs, int nrep,
                                       const int32_t* __restrict__ weight, const double* __restrict__ num_gt,
                                       const double* __restrict__ scores, const int32_t* __restrict__ frames,
                                       const int32_t* __restrict__ n_scores, double* __restrict__ thresholds,
                                       int32_t* __restrict__ n_thresh) {
    const long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (w >= njobs * nrep) return;
    const long long job = w / nrep;
    const int r = (int)(w % nrep);
    const Job jb = decode_job(e, job);
    const long long s0 = e.score_off[job], P = e.score_off[job + 1] - s0;
    const long long nj = n_scores[job] < P ? n_scores[job] : P;
    const int32_t* wr = weight + (long long)r * e.nframes;
    long long n = 0;
    for (long long i = 0; i < nj; ++i) n += wr[frames[s0 + i]];
    const double ngt = num_gt[(long long)r * e.nclass * e.ndiff + (long long)jb.c * e.ndiff + jb.d];
    const double step = 1.0 / (kThresh - 1.0);
    double* out = thresholds + ((long long)r * njobs + job) * kThresh;
    double cur = 0.0;
    int nt = 0;
    long long i = 0;
    for (long long q = 0; q < nj && nt < kThresh; ++q) {
        const int c = wr[frames[s0 + q]];
        const double sc = scores[s0 + q];
        for (int copy = 0; copy < c && nt < kThresh; ++copy, ++i) {
            const double l_recall = ddiv((double)(i + 1), ngt);
            const double r_recall = i < n - 1 ? ddiv((double)(i + 2), ngt) : l_recall;
            if (dsub(r_recall, cur) < dsub(cur, l_recall) && i < n - 1) continue;
            out[nt++] = sc;
            cur = dadd(cur, step);
        }
    }
    for (int t = nt; t < kThresh; ++t) out[t] = 0.0;
    n_thresh[(long long)r * njobs + job] = nt;
}

// Pass 2 of replicate r: one warp per (job, replicate), lane l at thresholds l and l + 32.  Each frame of the list
// list[list_off[r] .. list_off[r + 1]), in list order, adds the table entry of its smallest own score >= the
// threshold; the counts are integers (any order), the similarity is added in list order as fused_compute_statistics
// adds it over the frames.  A list may have any length (a drive-level replicate is longer or shorter than nframes).
constexpr int kBootWarps = 4;
__global__ void __launch_bounds__(32 * kBootWarps) boot_pr_kernel(SassdKittiEvalDesc e, long long njobs, int nrep,
                                                                  const int32_t* __restrict__ list,
                                                                  const int64_t* __restrict__ list_off,
                                                                  const double* __restrict__ thresholds,
                                                                  const int32_t* __restrict__ n_thresh,
                                                                  const int64_t* __restrict__ tab_off,
                                                                  const double* __restrict__ tab_score,
                                                                  const int32_t* __restrict__ tab_cnt,
                                                                  const double* __restrict__ tab_sim,
                                                                  const int32_t* __restrict__ tab_n,
                                                                  double* __restrict__ pr) {
    const long long wid = blockIdx.x * (long long)kBootWarps + threadIdx.x / 32;
    const int lane = threadIdx.x % 32;
    if (wid >= njobs * nrep) return;
    const long long job = wid / nrep;
    const int r = (int)(wid % nrep);
    const Job jb = decode_job(e, job);
    const bool aos = jb.m == 0 && e.aos_table && e.compute_aos[jb.k];
    const long long rj = (long long)r * njobs + job;
    const int nt = n_thresh[rj];
    constexpr int kPer = (kThresh + 31) / 32;
    double th[kPer], sim[kPer];
    long long tp[kPer], fp[kPer], fn[kPer];
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
        const int t = lane + 32 * u;
        th[u] = t < nt ? thresholds[rj * kThresh + t] : INFINITY;
        sim[u] = 0.0;
        tp[u] = fp[u] = fn[u] = 0;
    }
    if (lane < nt) {
        const long long p1 = list_off[r + 1];
        for (long long p = list_off[r]; p < p1; ++p) {
            const int f = list[p];
            const long long base = step_base(e, jb, job, tab_off, f);
            const int m = tab_n[job * e.nframes + f];
#pragma unroll
            for (int u = 0; u < kPer; ++u) {
                if (lane + 32 * u >= nt) break;
                int lo = 0, hi = m;                      // count the own scores >= th: entries 1..m descend
                while (lo < hi) {
                    const int mid = (lo + hi + 1) >> 1;
                    if (tab_score[base + mid] >= th[u]) lo = mid; else hi = mid - 1;
                }
                const long long at = base + lo;
                tp[u] += tab_cnt[3 * at];
                fp[u] += tab_cnt[3 * at + 1];
                fn[u] += tab_cnt[3 * at + 2];
                if (aos) {
                    const double s = tab_sim[at];
                    if (s != -1.0) sim[u] = dadd(sim[u], s);
                }
            }
        }
    }
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
        const int t = lane + 32 * u;
        if (t >= kThresh) break;
        double* o = pr + (rj * kThresh + t) * 4;
        o[0] = (double)tp[u];
        o[1] = (double)fp[u];
        o[2] = (double)fn[u];
        o[3] = sim[u];
    }
}

// The bootstrap's true-positive scores of each job sorted descending with their frames.  One CTA per job.
__global__ void boot_sort_kernel(SassdKittiEvalDesc e, double* __restrict__ scores, int32_t* __restrict__ frames,
                                 const int32_t* __restrict__ n_scores) {
    const long long job = blockIdx.x, s0 = e.score_off[job], P = e.score_off[job + 1] - s0;
    sort_desc(scores + s0, frames + s0, n_scores[job] < P ? n_scores[job] : P, P);
}

}  // namespace

extern "C" int sassd_kitti_eval_flags(int ngt, const int32_t* gt_name, const double* gt_occ, const double* gt_trunc,
                                      const double* gt_bbox, int ndt, const int32_t* dt_name, const double* dt_bbox,
                                      int nclass, const int32_t* classes, int ndiff, const double* limits,
                                      int8_t* ign_gt, int8_t* ign_dt, int32_t* n_valid, sassd_stream_t stream) {
    return sassd_kitti_eval_flags_ranged(ngt, gt_name, gt_occ, gt_trunc, gt_bbox, nullptr, ndt, dt_name, dt_bbox,
                                         nullptr, nclass, classes, ndiff, limits, nullptr, ign_gt, ign_dt, n_valid,
                                         nullptr, nullptr, stream);
}

extern "C" int sassd_kitti_eval_flags_ranged(int ngt, const int32_t* gt_name, const double* gt_occ,
                                             const double* gt_trunc, const double* gt_bbox, const double* gt_cam,
                                             int ndt, const int32_t* dt_name, const double* dt_bbox,
                                             const double* dt_cam, int nclass, const int32_t* classes, int ndiff,
                                             const double* limits, const double* ranges, int8_t* ign_gt,
                                             int8_t* ign_dt, int32_t* n_valid, double* gt_range, double* dt_range,
                                             sassd_stream_t stream) {
    if (ngt < 0 || ndt < 0 || nclass < 1 || ndiff < 1 || !classes || !limits || !n_valid) return SASSD_ERR_ARG;
    if (ngt > 0 && (!gt_name || !gt_occ || !gt_trunc || !gt_bbox || !ign_gt)) return SASSD_ERR_ARG;
    if (ndt > 0 && (!dt_name || !dt_bbox || !ign_dt)) return SASSD_ERR_ARG;
    if (ngt > 0 && (ranges || gt_range) && !gt_cam) return SASSD_ERR_ARG;
    if (ndt > 0 && (ranges || dt_range) && !dt_cam) return SASSD_ERR_ARG;
    const long long total = ((long long)ngt + ndt) * nclass * ndiff;
    if (total == 0) return SASSD_OK;
    eval_flags_kernel<<<sassd_grid(total, 256), 256, 0, (cudaStream_t)stream>>>(
        ngt, gt_name, gt_occ, gt_trunc, gt_bbox, gt_cam, ndt, dt_name, dt_bbox, dt_cam, nclass, classes, ndiff, limits,
        ranges, ign_gt, ign_dt, n_valid, gt_range, dt_range);
    return sassd_check_launch();
}

extern "C" int sassd_kitti_eval_overlaps(int nsets, int nframes, const int32_t* gt_off, const int32_t* dt_off,
                                         const int64_t* ov_off, const double* gt_cam, const double* dt_cam,
                                         const double* gt_bbox, const double* dt_bbox, const float* bev_iou,
                                         const float* bev_inter, int max_pairs_per_frame, double* ov_bbox,
                                         double* ov_bev, double* ov_3d, sassd_stream_t stream) {
    if (nsets < 1 || nframes < 0 || max_pairs_per_frame < 0 || !gt_off || !dt_off || !ov_off) return SASSD_ERR_ARG;
    if (nframes == 0 || max_pairs_per_frame == 0) return SASSD_OK;
    if (!gt_cam || !dt_cam || !gt_bbox || !dt_bbox || !bev_iou || !bev_inter || !ov_bbox || !ov_bev || !ov_3d)
        return SASSD_ERR_ARG;
    const long long blocks = (long long)nsets * nframes;
    dim3 grid((unsigned)sassd_div_up(max_pairs_per_frame, 128), (unsigned)(blocks < 32768 ? blocks : 32768));
    eval_overlaps_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(nsets, nframes, gt_off, dt_off,
                                                                 (const long long*)ov_off, gt_cam, dt_cam, gt_bbox,
                                                                 dt_bbox, bev_iou, bev_inter, ov_bbox, ov_bev, ov_3d);
    return sassd_check_launch();
}

extern "C" size_t sassd_kitti_eval_workspace_bytes(int max_nd, int max_ng) {
    if (max_nd < 0 || max_ng < 0) return 0;
    const size_t asg = ((size_t)kScratchThreads * (size_t)(max_nd > 0 ? max_nd : 1) + 255) / 256 * 256;
    return asg + (size_t)kScratchThreads * (size_t)(max_ng > 0 ? max_ng : 1) * sizeof(double);
}

extern "C" int sassd_kitti_eval_match(const SassdKittiEvalDesc* e, double* scores, int32_t* n_scores,
                                      double* thresholds, int32_t* n_thresh, double* pr, void* ws, size_t ws_bytes,
                                      sassd_stream_t stream_) {
    if (!e || e->nsets < 1 || e->nframes < 0 || e->nclass < 1 || e->ndiff < 1 || e->nover < 1 || e->max_nd < 0 ||
        e->max_ng < 0)
        return SASSD_ERR_ARG;
    const long long njobs = (long long)e->nsets * e->nclass * e->ndiff * 3 * e->nover;
    // one CTA per job sorts its scores; (job, threshold) items and job * frame items are counted in 64 bits
    if (njobs > 0x7fffffffLL || njobs * kThresh > 0x7fffffffLL) return SASSD_ERR_ARG;
    if (!e->gt_off || !e->dt_off || !e->ov_off || !e->gt_dc || !e->gt_bbox || !e->dt_bbox || !e->dt_score ||
        !e->ov_bbox || !e->ov_bev || !e->ov_3d || !e->compute_aos || !e->min_overlaps || !e->ign_gt || !e->ign_dt ||
        !e->n_valid || !e->score_off || !scores || !n_scores || !thresholds || !n_thresh || !pr || !ws)
        return SASSD_ERR_ARG;
    if (ws_bytes < sassd_kitti_eval_workspace_bytes(e->max_nd, e->max_ng)) return SASSD_ERR_WORKSPACE;
    cudaStream_t stream = (cudaStream_t)stream_;
    char* asg = (char*)ws;
    double* vals = (double*)(asg + ((size_t)kScratchThreads * (size_t)(e->max_nd > 0 ? e->max_nd : 1) + 255) / 256 * 256);
    if (cudaMemsetAsync(n_scores, 0, sizeof(int32_t) * njobs, stream) != cudaSuccess ||
        cudaMemsetAsync(n_thresh, 0, sizeof(int32_t) * njobs, stream) != cudaSuccess ||
        cudaMemsetAsync(pr, 0, sizeof(double) * 4 * kThresh * njobs, stream) != cudaSuccess)
        return SASSD_ERR_LAUNCH;
    if (e->nframes == 0) return SASSD_OK;
    eval_tp_scores_kernel<<<kMatchCtas, kMatchThreads, 0, stream>>>(*e, njobs, asg, scores, n_scores, nullptr);
    eval_thresholds_kernel<<<(unsigned)njobs, 1024, 0, stream>>>(*e, scores, n_scores, thresholds, n_thresh);
    eval_pr_kernel<<<kMatchCtas, kMatchThreads, 0, stream>>>(*e, njobs, asg, vals, thresholds, n_thresh, pr);
    return sassd_check_launch();
}

// Host function: the AOS term (1 + cos(gt alpha - dt alpha)) / 2 of every (detection, GT) pair, laid out like the
// overlap matrices, with the libm cos the host matcher (sassd_kitti_match) uses.
extern "C" int sassd_kitti_aos_table(int nsets, int nframes, const int32_t* gt_off, const int32_t* dt_off,
                                     const int64_t* ov_off, const double* gt_alpha, const double* dt_alpha, double* out) {
    if (nsets < 1 || nframes < 0 || !gt_off || !dt_off || !ov_off || !out) return SASSD_ERR_ARG;
    for (int b = 0; b < nsets * nframes; ++b) {
        const int f = b % nframes, g0 = gt_off[f], ng = gt_off[f + 1] - g0, d0 = dt_off[b], nd = dt_off[b + 1] - d0;
        double* o = out + ov_off[b];
        for (int j = 0; j < nd; ++j)
            for (int i = 0; i < ng; ++i) o[(size_t)j * ng + i] = (1.0 + std::cos(gt_alpha[g0 + i] - dt_alpha[d0 + j])) / 2.0;
    }
    return SASSD_OK;
}

extern "C" int sassd_kitti_eval_assign(const SassdKittiEvalDesc* e, int row, int ndiff, const double* gt_cam,
                                       const double* dt_cam, int32_t* gt_det, double* gt_ov, int8_t* dt_state,
                                       double* tp_err, void* ws, size_t ws_bytes, sassd_stream_t stream) {
    if (!e || e->nsets < 1 || e->nframes < 0 || e->nclass < 1 || e->ndiff < 1 || e->nover < 1 || e->max_nd < 0 ||
        e->max_ng < 0 || row < 0 || row >= e->nover || ndiff < 1 || ndiff > e->ndiff)
        return SASSD_ERR_ARG;
    if (!e->gt_off || !e->dt_off || !e->ov_off || !e->gt_dc || !e->gt_bbox || !e->dt_bbox || !e->dt_score ||
        !e->ov_bbox || !e->ov_bev || !e->ov_3d || !e->min_overlaps || !e->ign_gt || !e->ign_dt || !gt_cam || !dt_cam ||
        !gt_det || !gt_ov || !dt_state || !tp_err || !ws)
        return SASSD_ERR_ARG;
    if (ws_bytes < sassd_kitti_eval_workspace_bytes(e->max_nd, e->max_ng)) return SASSD_ERR_WORKSPACE;
    if (e->nframes == 0) return SASSD_OK;
    const long long njobs = (long long)e->nsets * e->nclass * ndiff * 3;
    eval_assign_kernel<<<kMatchCtas, kMatchThreads, 0, (cudaStream_t)stream>>>(*e, row, ndiff, njobs, (char*)ws, gt_cam,
                                                                             dt_cam, gt_det, gt_ov, dt_state, tp_err);
    return sassd_check_launch();
}

static bool boot_desc_ok(const SassdKittiEvalDesc* e) {
    return e && e->nsets >= 1 && e->nframes >= 1 && e->nclass >= 1 && e->ndiff >= 1 && e->nover >= 1 &&
           e->max_nd >= 0 && e->max_ng >= 0 && e->gt_off && e->dt_off && e->ov_off && e->gt_dc && e->gt_bbox &&
           e->dt_bbox && e->dt_score && e->ov_bbox && e->ov_bev && e->ov_3d && e->compute_aos && e->min_overlaps &&
           e->ign_gt && e->ign_dt && e->n_valid && e->score_off;
}

extern "C" int sassd_kitti_boot_prepare(const SassdKittiEvalDesc* e, double* scores, int32_t* frames,
                                        int32_t* n_scores, const int64_t* tab_off, double* tab_score,
                                        int32_t* tab_cnt, double* tab_sim, int32_t* tab_n, void* ws, size_t ws_bytes,
                                        sassd_stream_t stream_) {
    if (!boot_desc_ok(e) || !scores || !frames || !n_scores || !tab_off || !tab_score || !tab_cnt || !tab_sim ||
        !tab_n || !ws)
        return SASSD_ERR_ARG;
    const long long njobs = (long long)e->nsets * e->nclass * e->ndiff * 3 * e->nover;
    if (njobs > 0x7fffffffLL) return SASSD_ERR_ARG;
    if (ws_bytes < sassd_kitti_eval_workspace_bytes(e->max_nd, e->max_ng)) return SASSD_ERR_WORKSPACE;
    cudaStream_t stream = (cudaStream_t)stream_;
    char* asg = (char*)ws;
    double* vals = (double*)(asg + ((size_t)kScratchThreads * (size_t)(e->max_nd > 0 ? e->max_nd : 1) + 255) / 256 * 256);
    if (cudaMemsetAsync(n_scores, 0, sizeof(int32_t) * njobs, stream) != cudaSuccess) return SASSD_ERR_LAUNCH;
    eval_tp_scores_kernel<<<kMatchCtas, kMatchThreads, 0, stream>>>(*e, njobs, asg, scores, n_scores, frames);
    boot_sort_kernel<<<(unsigned)njobs, 1024, 0, stream>>>(*e, scores, frames, n_scores);
    boot_steps_kernel<<<kMatchCtas, kMatchThreads, 0, stream>>>(*e, njobs, asg, vals, tab_off, tab_score, tab_cnt,
                                                                tab_sim, tab_n);
    return sassd_check_launch();
}

extern "C" int sassd_kitti_boot_eval(const SassdKittiEvalDesc* e, int nrep, const int32_t* list,
                                     const int64_t* list_off, const int32_t* weight, const double* num_gt,
                                     const double* scores, const int32_t* frames, const int32_t* n_scores,
                                     const int64_t* tab_off, const double* tab_score, const int32_t* tab_cnt,
                                     const double* tab_sim, const int32_t* tab_n, double* thresholds,
                                     int32_t* n_thresh, double* pr, sassd_stream_t stream_) {
    if (!boot_desc_ok(e) || nrep < 1 || !list || !list_off || !weight || !num_gt || !scores || !frames || !n_scores ||
        !tab_off || !tab_score || !tab_cnt || !tab_sim || !tab_n || !thresholds || !n_thresh || !pr)
        return SASSD_ERR_ARG;
    const long long njobs = (long long)e->nsets * e->nclass * e->ndiff * 3 * e->nover;
    const long long items = njobs * nrep;
    if (njobs > 0x7fffffffLL || items > 0x7fffffffLL * (long long)kBootWarps) return SASSD_ERR_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    boot_thresholds_kernel<<<(unsigned)sassd_div_up(items, 128), 128, 0, stream>>>(
        *e, njobs, nrep, weight, num_gt, scores, frames, n_scores, thresholds, n_thresh);
    boot_pr_kernel<<<(unsigned)sassd_div_up(items, kBootWarps), 32 * kBootWarps, 0, stream>>>(
        *e, njobs, nrep, list, list_off, thresholds, n_thresh, tab_off, tab_score, tab_cnt, tab_sim, tab_n, pr);
    return sassd_check_launch();
}

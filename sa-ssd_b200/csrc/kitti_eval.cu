// KITTI evaluation support (SURVEY.md section 8, row f4):
//  * rotated-box overlap for the BEV / 3-D metrics as a batched CUDA kernel — the reference runs this step as
//    numba.cuda code (mmdet/core/post_processing/rotate_nms_gpu.py:153-381 geometry, :536-548 criteria,
//    :551-627 launch), one launch per 1/50th of the dataset; here one launch covers every frame;
//  * the greedy GT<->detection matching and the per-threshold tp/fp/fn/similarity accumulation
//    (mmdet/core/evaluation/kitti_eval.py:164-283 compute_statistics_jit, :295-342 fused_compute_statistics) as host
//    code — numba-jitted CPU code in the reference, plain C++ here (no GPU needed for this part).
// The float32 geometry is written with round-to-nearest intrinsics and no FMA contraction so that it reproduces the
// reference's operation sequence bit for bit (oracle/kitti_eval.py, pinned on tests/golden/eval.npz).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

#include "common.cuh"

namespace {

struct P2f { float x, y; };

__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float dvd(float a, float b) { return __fdiv_rn(a, b); }

// clockwise corners rotated clockwise by the angle (rotate_nms_gpu.py:340-363)
__device__ void box_corners(const float* b, P2f* c) {
    const float cs = (float)cos((double)b[4]), sn = (float)sin((double)b[4]);
    const float hx = dvd(b[2], 2.f), hy = dvd(b[3], 2.f);
    const float xs[4] = {-hx, -hx, hx, hx}, ys[4] = {-hy, hy, hy, -hy};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        c[i].x = add(add(mul(cs, xs[i]), mul(sn, ys[i])), b[0]);
        c[i].y = add(add(mul(-sn, xs[i]), mul(cs, ys[i])), b[1]);
    }
}

// :297-313
__device__ bool inside(float px, float py, const P2f* q) {
    const float ab0 = sub(q[1].x, q[0].x), ab1 = sub(q[1].y, q[0].y);
    const float ad0 = sub(q[3].x, q[0].x), ad1 = sub(q[3].y, q[0].y);
    const float ap0 = sub(px, q[0].x), ap1 = sub(py, q[0].y);
    const float abab = add(mul(ab0, ab0), mul(ab1, ab1)), abap = add(mul(ab0, ap0), mul(ab1, ap1));
    const float adad = add(mul(ad0, ad0), mul(ad1, ad1)), adap = add(mul(ad0, ap0), mul(ad1, ap1));
    return abab >= abap && abap >= 0.f && adad >= adap && adap >= 0.f;
}

// edge i of p1 against edge j of p2 (:209-252)
__device__ bool segment_hit(const P2f* p1, const P2f* p2, int i, int j, P2f* out) {
    const P2f a = p1[i], b = p1[(i + 1) & 3], c = p2[j], d = p2[(j + 1) & 3];
    const float ba0 = sub(b.x, a.x), ba1 = sub(b.y, a.y);
    const float da0 = sub(d.x, a.x), ca0 = sub(c.x, a.x), da1 = sub(d.y, a.y), ca1 = sub(c.y, a.y);
    const bool acd = mul(da1, ca0) > mul(ca1, da0);
    const bool bcd = mul(sub(d.y, b.y), sub(c.x, b.x)) > mul(sub(c.y, b.y), sub(d.x, b.x));
    if (acd == bcd) return false;
    const bool abc = mul(ca1, ba0) > mul(ba1, ca0), abd = mul(da1, ba0) > mul(ba1, da0);
    if (abc == abd) return false;
    const float dc0 = sub(d.x, c.x), dc1 = sub(d.y, c.y);
    const float abba = sub(mul(a.x, b.y), mul(b.x, a.y)), cddc = sub(mul(c.x, d.y), mul(d.x, c.y));
    const float dh = sub(mul(ba1, dc0), mul(ba0, dc1));
    out->x = dvd(sub(mul(abba, dc0), mul(ba0, cddc)), dh);
    out->y = dvd(sub(mul(abba, dc1), mul(ba1, cddc)), dh);
    return true;
}

// Intersection area of the quadrilaterals p1 and p2 by Sutherland-Hodgman clipping of p1 against p2's edges in fp64,
// rounded to float and clamped to [0, amin].  Used only where the reference's result is undefined (see pts[24]
// below).  A convex input gives at most 8 vertices; the 16-entry buffers only bound what rounding can add.
__device__ float clipped_area(const P2f* p1, const P2f* p2, float amin) {
    double sx[16], sy[16], tx[16], ty[16], d[16];
    int n = 4;
    for (int i = 0; i < 4; ++i) { sx[i] = p1[i].x; sy[i] = p1[i].y; }
    double s2 = 0.0;      // twice p2's signed area: the side its interior is on
    for (int i = 0; i < 4; ++i) {
        const int k = (i + 1) & 3;
        s2 = __dadd_rn(s2, __dsub_rn(__dmul_rn(p2[i].x, p2[k].y), __dmul_rn(p2[k].x, p2[i].y)));
    }
    if (!(s2 != 0.0)) return 0.f;
    const double sg = s2 > 0.0 ? 1.0 : -1.0;
    for (int e = 0; e < 4 && n > 0; ++e) {
        const double ax = p2[e].x, ay = p2[e].y;
        const double ex = __dsub_rn(p2[(e + 1) & 3].x, ax), ey = __dsub_rn(p2[(e + 1) & 3].y, ay);
        for (int i = 0; i < n; ++i)
            d[i] = sg * __dsub_rn(__dmul_rn(ex, __dsub_rn(sy[i], ay)), __dmul_rn(ey, __dsub_rn(sx[i], ax)));
        int m = 0;
        for (int i = 0; i < n; ++i) {
            const int k = i + 1 == n ? 0 : i + 1;
            if (d[i] >= 0.0 && m < 16) { tx[m] = sx[i]; ty[m] = sy[i]; ++m; }
            if ((d[i] >= 0.0) != (d[k] >= 0.0) && m < 16) {
                const double t = __ddiv_rn(d[i], __dsub_rn(d[i], d[k]));
                tx[m] = __dadd_rn(sx[i], __dmul_rn(t, __dsub_rn(sx[k], sx[i])));
                ty[m] = __dadd_rn(sy[i], __dmul_rn(t, __dsub_rn(sy[k], sy[i])));
                ++m;
            }
        }
        for (int i = 0; i < m; ++i) { sx[i] = tx[i]; sy[i] = ty[i]; }
        n = m;
    }
    double a = 0.0;
    for (int i = 0; i < n; ++i) {
        const int k = i + 1 == n ? 0 : i + 1;
        a = __dadd_rn(a, __dsub_rn(__dmul_rn(sx[i], sy[k]), __dmul_rn(sx[k], sy[i])));
    }
    const float r = __double2float_rn(__dmul_rn(fabs(a), 0.5));
    return r < amin ? r : amin;
}

// area of the intersection polygon of two rotated boxes (x, y, dx, dy, angle) (:366-380)
__device__ float rotated_intersection(const float* b1, const float* b2) {
    // The reference collects the points into a 16-float local array, 8 points.  Where edges of the two boxes
    // coincide up to rounding (a box against itself turned by pi, or by 1e-7) nearly parallel edges pass its
    // crossing tests and it collects up to 24 points (8 corners, 16 hits): it writes past its array, so its value
    // there is undefined, and its own arithmetic on those points gives intersections above the boxes' areas.
    // pts[24] holds every point the collection can make.  Up to 8 points the result is the reference's, bit for
    // bit; past 8 it is clipped_area's, which is within 2^-24 A + 2^-40 (M + 1)^2 of min(A, amin), A the exact
    // intersection of the same float corners, M their largest |coordinate| and amin the smaller |dx * dy|; it never
    // exceeds amin and is never negative or NaN for finite boxes (tests/test_kitti_eval_geometry.py).
    P2f p1[4], p2[4], pts[24];
    box_corners(b1, p1);
    box_corners(b2, p2);
    int n = 0;
    for (int i = 0; i < 4; ++i) {
        if (inside(p1[i].x, p1[i].y, p2)) pts[n++] = p1[i];
        if (inside(p2[i].x, p2[i].y, p1)) pts[n++] = p2[i];
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            P2f h;
            if (segment_hit(p1, p2, i, j, &h)) pts[n++] = h;
        }
    if (n > 8) return clipped_area(p1, p2, fminf(fabsf(mul(b1[2], b1[3])), fabsf(mul(b2[2], b2[3]))));
    if (n > 0) {      // sort by a monotone key of the polar angle about the centroid (:169-206)
        float cx = 0.f, cy = 0.f;
        for (int i = 0; i < n; ++i) { cx = add(cx, pts[i].x); cy = add(cy, pts[i].y); }
        cx = dvd(cx, (float)n);
        cy = dvd(cy, (float)n);
        float key[24];
        for (int i = 0; i < n; ++i) {
            float vx = sub(pts[i].x, cx), vy = sub(pts[i].y, cy);
            const float d = __fsqrt_rn(add(mul(vx, vx), mul(vy, vy)));
            vx = dvd(vx, d);
            vy = dvd(vy, d);
            key[i] = vy < 0.f ? sub(-2.f, vx) : vx;
        }
        for (int i = 1; i < n; ++i)
            if (key[i - 1] > key[i]) {
                const float tk = key[i];
                const P2f tp = pts[i];
                int j = i;
                while (j > 0 && key[j - 1] > tk) { key[j] = key[j - 1]; pts[j] = pts[j - 1]; --j; }
                key[j] = tk;
                pts[j] = tp;
            }
    }
    float area = 0.f;      // triangle fan about the first vertex (:153-166)
    for (int i = 0; i + 2 < n; ++i) {
        const P2f a = pts[0], b = pts[i + 1], c = pts[i + 2];
        const float t = dvd(sub(mul(sub(a.x, c.x), sub(b.y, c.y)), mul(sub(a.y, c.y), sub(b.x, c.x))), 2.f);
        area = add(area, fabsf(t));
    }
    return area;
}

// One thread per (box, query) pair of one frame; frames are ranges of the concatenated arrays.
__global__ void rotate_overlap_eval_kernel(const float* __restrict__ boxes, const int* __restrict__ box_off,
                                           const float* __restrict__ query, const int* __restrict__ query_off,
                                           const long long* __restrict__ out_off, int nframes, int criterion,
                                           float* __restrict__ out) {
    for (int f = blockIdx.y; f < nframes; f += gridDim.y) {
        const int nb = box_off[f + 1] - box_off[f], nq = query_off[f + 1] - query_off[f];
        const long long total = (long long)nb * nq;
        for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
             i += (long long)gridDim.x * blockDim.x) {
            const int n = (int)(i / nq), k = (int)(i % nq);
            const float* b = boxes + (size_t)(box_off[f] + n) * 5;
            const float* q = query + (size_t)(query_off[f] + k) * 5;
            // the reference passes the QUERY box first (:586-588): criterion 0 divides by its area
            const float a1 = mul(q[2], q[3]), a2 = mul(b[2], b[3]);
            const float it = rotated_intersection(q, b);
            float v;
            if (criterion == -1) v = dvd(it, sub(add(a1, a2), it));
            else if (criterion == 0) v = dvd(it, a1);
            else if (criterion == 1) v = dvd(it, a2);
            else v = it;
            out[out_off[f] + i] = v;
        }
    }
}

// kitti_eval.py:95-122 with criterion 0 (intersection over the first box's area), one detection x one DontCare box
inline double box_overlap_first(const double* b, const double* q) {
    const double iw = std::min(b[2], q[2]) - std::max(b[0], q[0]);
    if (iw <= 0) return 0.0;
    const double ih = std::min(b[3], q[3]) - std::max(b[1], q[1]);
    if (ih <= 0) return 0.0;
    return iw * ih / ((b[2] - b[0]) * (b[3] - b[1]));
}

struct FrameView {
    const double* ov;      // [nd, ng]
    int ng, nd, ndc;
    const double *gt_alpha, *dt_alpha, *dt_score, *dt_bbox, *dc_bbox;
    const int32_t *ign_gt, *ign_dt;
};

// Where frame_statistics records its assignment (sassd_kitti_assign): per GT row the matched detection's row (row0 +
// its index in the frame) or -1 and their overlap, per detection its SASSD_KITTI_DT_* state.
struct AssignRecord {
    int32_t* gt_det;
    double* gt_ov;
    int8_t* dt_state;
    int row0;
};

// compute_statistics_jit (:164-283).  Returns tp; fills fp, fn, similarity; appends TP scores when asked; records the
// assignment when `rec` is given.
int frame_statistics(const FrameView& f, int metric, double min_overlap, double thresh, bool compute_fp, bool compute_aos,
                     int* fp_out, int* fn_out, double* sim_out, double* tp_scores, long long* n_tp_scores,
                     std::vector<char>& assigned, std::vector<char>& below, std::vector<double>& delta,
                     const AssignRecord* rec = nullptr) {
    if (rec) {
        for (int i = 0; i < f.ng; ++i) { rec->gt_det[i] = -1; rec->gt_ov[i] = 0.0; }
        for (int j = 0; j < f.nd; ++j) rec->dt_state[j] = SASSD_KITTI_DT_NOT_COUNTED;
    }
    assigned.assign(f.nd, 0);
    below.assign(f.nd, 0);
    delta.clear();
    if (compute_fp)
        for (int j = 0; j < f.nd; ++j) below[j] = f.dt_score[j] < thresh;
    const double NO = -10000000;
    int tp = 0, fp = 0, fn = 0;
    for (int i = 0; i < f.ng; ++i) {
        if (f.ign_gt[i] == -1) continue;
        int det = -1;
        double valid = NO, max_ov = 0;
        bool assigned_ign = false;
        for (int j = 0; j < f.nd; ++j) {
            if (f.ign_dt[j] == -1 || assigned[j] || below[j]) continue;
            const double ov = f.ov[(size_t)j * f.ng + i];
            if (!compute_fp && ov > min_overlap && f.dt_score[j] > valid) {
                det = j; valid = f.dt_score[j];
            } else if (compute_fp && ov > min_overlap && (ov > max_ov || assigned_ign) && f.ign_dt[j] == 0) {
                max_ov = ov; det = j; valid = 1; assigned_ign = false;
            } else if (compute_fp && ov > min_overlap && valid == NO && f.ign_dt[j] == 1) {
                det = j; valid = 1; assigned_ign = true;
            }
        }
        if (valid == NO && f.ign_gt[i] == 0) {
            ++fn;
        } else if (valid != NO && (f.ign_gt[i] == 1 || f.ign_dt[det] == 1)) {
            assigned[det] = 1;
            if (rec) rec->dt_state[det] = SASSD_KITTI_DT_IGNORED;
        } else if (valid != NO) {
            ++tp;
            if (tp_scores) tp_scores[(*n_tp_scores)++] = f.dt_score[det];
            if (compute_aos) delta.push_back(f.gt_alpha[i] - f.dt_alpha[det]);
            assigned[det] = 1;
            if (rec) rec->dt_state[det] = SASSD_KITTI_DT_TP;
        }
        if (rec && valid != NO) {
            rec->gt_det[i] = rec->row0 + det;
            rec->gt_ov[i] = f.ov[(size_t)det * f.ng + i];
        }
    }
    double similarity = 0;
    if (compute_fp) {
        for (int j = 0; j < f.nd; ++j)
            if (!(assigned[j] || f.ign_dt[j] == -1 || f.ign_dt[j] == 1 || below[j])) {
                ++fp;
                if (rec) rec->dt_state[j] = SASSD_KITTI_DT_FP;
            }
        int nstuff = 0;
        if (metric == 0)
            for (int i = 0; i < f.ndc; ++i)
                for (int j = 0; j < f.nd; ++j) {
                    if (assigned[j] || f.ign_dt[j] == -1 || f.ign_dt[j] == 1 || below[j]) continue;
                    if (box_overlap_first(f.dt_bbox + 4 * (size_t)j, f.dc_bbox + 4 * (size_t)i) > min_overlap) {
                        assigned[j] = 1;
                        ++nstuff;
                        if (rec) rec->dt_state[j] = SASSD_KITTI_DT_DONTCARE;
                    }
                }
        fp -= nstuff;
        if (compute_aos) {
            if (tp > 0 || fp > 0) {
                // np.sum over [zeros(fp), (1 + cos(delta)) / 2 ...]: numpy's pairwise summation order
                std::vector<double> tmp((size_t)std::max(fp, 0) + delta.size(), 0.0);
                for (size_t i = 0; i < delta.size(); ++i) tmp[(size_t)std::max(fp, 0) + i] = (1.0 + std::cos(delta[i])) / 2.0;
                struct Pairwise {
                    static double sum(const double* a, size_t n) {
                        if (n < 8) { double s = 0; for (size_t i = 0; i < n; ++i) s += a[i]; return s; }
                        if (n <= 128) {
                            double r[8];
                            for (int k = 0; k < 8; ++k) r[k] = a[k];
                            size_t i = 8;
                            for (; i + 8 <= n; i += 8) for (int k = 0; k < 8; ++k) r[k] += a[i + k];
                            double s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
                            for (; i < n; ++i) s += a[i];
                            return s;
                        }
                        size_t n2 = n / 2;
                        n2 -= n2 % 8;
                        return sum(a, n2) + sum(a + n2, n - n2);
                    }
                };
                similarity = Pairwise::sum(tmp.data(), tmp.size());
            } else {
                similarity = -1;
            }
        }
    }
    *fp_out = fp; *fn_out = fn; *sim_out = similarity;
    return tp;
}

}  // namespace

extern "C" int sassd_rotate_overlap_eval(const float* boxes, const int32_t* box_off, const float* query,
                                         const int32_t* query_off, const int64_t* out_off, int nframes, int criterion,
                                         int max_pairs_per_frame, float* out, sassd_stream_t stream_) {
    if (!boxes || !box_off || !query || !query_off || !out_off || !out || nframes < 0) return SASSD_ERR_ARG;
    if (criterion < -1 || criterion > 2) return SASSD_ERR_ARG;
    if (nframes == 0 || max_pairs_per_frame <= 0) return SASSD_OK;
    dim3 grid((unsigned)sassd_div_up(max_pairs_per_frame, 128), (unsigned)(nframes < 32768 ? nframes : 32768));
    rotate_overlap_eval_kernel<<<grid, 128, 0, (cudaStream_t)stream_>>>(boxes, box_off, query, query_off,
                                                                        (const long long*)out_off, nframes, criterion, out);
    return sassd_check_launch();
}

// Host function (no GPU involved).  Frame f owns gt rows [gt_off[f], gt_off[f+1]), detection rows
// [dt_off[f], dt_off[f+1]), DontCare boxes [dc_off[f], dc_off[f+1]) and the row-major overlap block
// overlaps[ov_off[f] + j * ng_f + i] (detection j, ground truth i).
// nthresh == 0: matching pass without false positives (compute_fp=False): appends the scores of the true positives
// to tp_scores (capacity = total gt rows) and sets *n_tp_scores.  nthresh > 0: for every threshold accumulate
// pr[t] += (tp, fp, fn, similarity) over all frames (fused_compute_statistics).
extern "C" int sassd_kitti_match(int nframes, const double* overlaps, const int64_t* ov_off, const int32_t* gt_off,
                                 const int32_t* dt_off, const int32_t* dc_off, const double* gt_alpha,
                                 const double* dt_alpha, const double* dt_score, const double* dt_bbox,
                                 const double* dc_bbox, const int32_t* ign_gt, const int32_t* ign_dt, int metric,
                                 double min_overlap, int compute_aos, int nthresh, const double* thresholds, double* pr,
                                 double* tp_scores, int64_t* n_tp_scores) {
    if (nframes < 0 || !ov_off || !gt_off || !dt_off || !dc_off || metric < 0 || metric > 2) return SASSD_ERR_ARG;
    if (nthresh == 0 && (!tp_scores || !n_tp_scores)) return SASSD_ERR_ARG;
    if (nthresh > 0 && (!thresholds || !pr)) return SASSD_ERR_ARG;
    std::vector<char> assigned, below;
    std::vector<double> delta;
    long long ntp = 0;
    for (int f = 0; f < nframes; ++f) {
        FrameView v;
        v.ng = gt_off[f + 1] - gt_off[f]; v.nd = dt_off[f + 1] - dt_off[f]; v.ndc = dc_off[f + 1] - dc_off[f];
        v.ov = overlaps + ov_off[f];
        v.gt_alpha = gt_alpha + gt_off[f]; v.dt_alpha = dt_alpha + dt_off[f]; v.dt_score = dt_score + dt_off[f];
        v.dt_bbox = dt_bbox + 4 * (size_t)dt_off[f]; v.dc_bbox = dc_bbox + 4 * (size_t)dc_off[f];
        v.ign_gt = ign_gt + gt_off[f]; v.ign_dt = ign_dt + dt_off[f];
        int fp, fn;
        double sim;
        if (nthresh == 0) {
            frame_statistics(v, metric, min_overlap, 0.0, false, false, &fp, &fn, &sim, tp_scores, &ntp, assigned, below,
                             delta);
        } else {
            for (int t = 0; t < nthresh; ++t) {
                const int tp = frame_statistics(v, metric, min_overlap, thresholds[t], true, compute_aos != 0, &fp, &fn,
                                                &sim, nullptr, nullptr, assigned, below, delta);
                pr[4 * t + 0] += tp; pr[4 * t + 1] += fp; pr[4 * t + 2] += fn;
                if (sim != -1) pr[4 * t + 3] += sim;
            }
        }
    }
    if (n_tp_scores) *n_tp_scores = ntp;
    return SASSD_OK;
}

// Host function: frame_statistics' assignment at a threshold below every score, recorded frame by frame.
extern "C" int sassd_kitti_assign(int nframes, const double* overlaps, const int64_t* ov_off, const int32_t* gt_off,
                                  const int32_t* dt_off, const int32_t* dc_off, const double* dt_score,
                                  const double* dt_bbox, const double* dc_bbox, const int32_t* ign_gt,
                                  const int32_t* ign_dt, int metric, double min_overlap, int32_t* gt_det, double* gt_ov,
                                  int8_t* dt_state) {
    if (nframes < 0 || !ov_off || !gt_off || !dt_off || !dc_off || metric < 0 || metric > 2) return SASSD_ERR_ARG;
    if (nframes > 0 && (gt_off[nframes] > 0 && (!gt_det || !gt_ov || !ign_gt))) return SASSD_ERR_ARG;
    if (nframes > 0 && (dt_off[nframes] > 0 && (!dt_state || !ign_dt || !dt_score || !dt_bbox))) return SASSD_ERR_ARG;
    std::vector<char> assigned, below;
    std::vector<double> delta;
    for (int f = 0; f < nframes; ++f) {
        FrameView v;
        v.ng = gt_off[f + 1] - gt_off[f]; v.nd = dt_off[f + 1] - dt_off[f]; v.ndc = dc_off[f + 1] - dc_off[f];
        v.ov = overlaps + ov_off[f];
        v.gt_alpha = nullptr; v.dt_alpha = nullptr; v.dt_score = dt_score + dt_off[f];
        v.dt_bbox = dt_bbox + 4 * (size_t)dt_off[f]; v.dc_bbox = dc_bbox + 4 * (size_t)dc_off[f];
        v.ign_gt = ign_gt + gt_off[f]; v.ign_dt = ign_dt + dt_off[f];
        AssignRecord rec{gt_det + gt_off[f], gt_ov + gt_off[f], dt_state + dt_off[f], dt_off[f]};
        int fp, fn;
        double sim;
        frame_statistics(v, metric, min_overlap, -INFINITY, true, false, &fp, &fn, &sim, nullptr, nullptr, assigned,
                         below, delta, &rec);
    }
    return SASSD_OK;
}

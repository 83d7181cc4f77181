/* ORACLE — test infrastructure only (see oracle/voxelize.c header).
 *
 * CPU restatement of the reference rotated-BEV NMS:
 *   mmdet/ops/iou3d/src/iou3d_kernel.cu:34-106  (cross products, segment
 *        intersection, point-in-rotated-box with 1e-5 margin)
 *   mmdet/ops/iou3d/src/iou3d_kernel.cu:108-212 (box_overlap: corner rotation,
 *        16 edge intersections, contained corners, bubble sort by atan2 about
 *        the centroid, fan-triangulated shoelace area)
 *   mmdet/ops/iou3d/src/iou3d_kernel.cu:214-221 (iou_bev, eps 1e-8)
 *   mmdet/ops/iou3d/src/iou3d_kernel.cu:250-292 (64x64 tiled suppression bitmask,
 *        strict '>' threshold, j > i only inside the diagonal tile)
 *   mmdet/ops/iou3d/src/iou3d.cpp:100-116       (greedy sweep over the bitmask)
 *   mmdet/ops/iou3d/iou3d_utils.py:114-128      (sort by score, descending)
 *
 * The reference source is CUDA-only; on the GPU box the unmodified reference
 * kernel (oracle/_ref/libiou3d_ref.so, built by oracle/build.py from
 * /root/reference in place) pins the bitmask bit-for-bit.  This C version is
 * the CPU checker; it evaluates in fp32 without FMA contraction, so an IoU
 * that lands within a few ulp of the threshold may differ from the GPU — the
 * tests report min |IoU - thr| next to every keep-mask comparison.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float x, y; } pt_t;

static const float kEps = 1e-8f;

static inline float cross2(pt_t a, pt_t b) { return a.x * b.y - a.y * b.x; }

static inline float cross3(pt_t p1, pt_t p2, pt_t p0)
{
    return (p1.x - p0.x) * (p2.y - p0.y) - (p2.x - p0.x) * (p1.y - p0.y);
}

static inline int bbox_disjoint_test(pt_t p1, pt_t p2, pt_t q1, pt_t q2)
{
    return fminf(p1.x, p2.x) <= fmaxf(q1.x, q2.x) && fminf(q1.x, q2.x) <= fmaxf(p1.x, p2.x) &&
           fminf(p1.y, p2.y) <= fmaxf(q1.y, q2.y) && fminf(q1.y, q2.y) <= fmaxf(p1.y, p2.y);
}

/* box = [x1, y1, x2, y2, angle] */
static inline int inside_box(const float *box, pt_t p)
{
    const float margin = 1e-5f;
    float cx = (box[0] + box[2]) / 2, cy = (box[1] + box[3]) / 2;
    float c = cosf(-box[4]), s = sinf(-box[4]);
    float rx = (p.x - cx) * c + (p.y - cy) * s + cx;
    float ry = -(p.x - cx) * s + (p.y - cy) * c + cy;
    return rx > box[0] - margin && rx < box[2] + margin && ry > box[1] - margin && ry < box[3] + margin;
}

static inline int seg_intersect(pt_t p1, pt_t p0, pt_t q1, pt_t q0, pt_t *ans)
{
    if (!bbox_disjoint_test(p0, p1, q0, q1)) return 0;
    float s1 = cross3(q0, p1, p0);
    float s2 = cross3(p1, q1, p0);
    float s3 = cross3(p0, q1, q0);
    float s4 = cross3(q1, p1, q0);
    if (!(s1 * s2 > 0 && s3 * s4 > 0)) return 0;
    float s5 = cross3(q1, p1, p0);
    if (fabsf(s5 - s1) > kEps) {
        ans->x = (s5 * q0.x - s1 * q1.x) / (s5 - s1);
        ans->y = (s5 * q0.y - s1 * q1.y) / (s5 - s1);
    } else {
        float a0 = p0.y - p1.y, b0 = p1.x - p0.x, c0 = p0.x * p1.y - p1.x * p0.y;
        float a1 = q0.y - q1.y, b1 = q1.x - q0.x, c1 = q0.x * q1.y - q1.x * q0.y;
        float D = a0 * b1 - a1 * b0;
        ans->x = (b0 * c1 - b1 * c0) / D;
        ans->y = (a1 * c0 - a0 * c1) / D;
    }
    return 1;
}

static inline pt_t rot_about(pt_t ctr, float c, float s, pt_t p)
{
    pt_t r;
    r.x = (p.x - ctr.x) * c + (p.y - ctr.y) * s + ctr.x;
    r.y = -(p.x - ctr.x) * s + (p.y - ctr.y) * c + ctr.y;
    return r;
}

/* The reference keeps 16 polygon points; this restatement has room for every point the loops can add (16 edge
 * hits and 8 corners) so that it can report a pair that would need more (*count), without writing out of bounds. */
static float box_overlap_count(const float *a, const float *b, int *count)
{
    pt_t ca = { (a[0] + a[2]) / 2, (a[1] + a[3]) / 2 };
    pt_t cb = { (b[0] + b[2]) / 2, (b[1] + b[3]) / 2 };
    pt_t A[5] = { {a[0], a[1]}, {a[2], a[1]}, {a[2], a[3]}, {a[0], a[3]} };
    pt_t B[5] = { {b[0], b[1]}, {b[2], b[1]}, {b[2], b[3]}, {b[0], b[3]} };
    float cas = cosf(a[4]), sas = sinf(a[4]);
    float cbs = cosf(b[4]), sbs = sinf(b[4]);
    for (int k = 0; k < 4; ++k) {
        A[k] = rot_about(ca, cas, sas, A[k]);
        B[k] = rot_about(cb, cbs, sbs, B[k]);
    }
    A[4] = A[0];
    B[4] = B[0];

    pt_t poly[24];
    pt_t ctr = { 0.f, 0.f };
    int cnt = 0;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            if (seg_intersect(A[i + 1], A[i], B[j + 1], B[j], &poly[cnt])) {
                ctr.x = ctr.x + poly[cnt].x;
                ctr.y = ctr.y + poly[cnt].y;
                ++cnt;
            }
    for (int k = 0; k < 4; ++k) {
        if (inside_box(a, B[k])) {
            ctr.x = ctr.x + B[k].x; ctr.y = ctr.y + B[k].y;
            poly[cnt++] = B[k];
        }
        if (inside_box(b, A[k])) {
            ctr.x = ctr.x + A[k].x; ctr.y = ctr.y + A[k].y;
            poly[cnt++] = A[k];
        }
    }
    *count = cnt;
    ctr.x /= cnt;
    ctr.y /= cnt;
    /* bubble sort, ascending polar angle about the centroid (iou3d_kernel.cu:183-193) */
    for (int j = 0; j < cnt - 1; ++j)
        for (int i = 0; i < cnt - j - 1; ++i)
            if (atan2f(poly[i].y - ctr.y, poly[i].x - ctr.x) >
                atan2f(poly[i + 1].y - ctr.y, poly[i + 1].x - ctr.x)) {
                pt_t t = poly[i]; poly[i] = poly[i + 1]; poly[i + 1] = t;
            }
    float area = 0;
    for (int k = 0; k < cnt - 1; ++k) {
        pt_t u = { poly[k].x - poly[0].x, poly[k].y - poly[0].y };
        pt_t v = { poly[k + 1].x - poly[0].x, poly[k + 1].y - poly[0].y };
        area += cross2(u, v);
    }
    return fabsf(area) / 2.0f;
}

float oracle_box_overlap(const float *a, const float *b)
{
    int cnt;
    return box_overlap_count(a, b, &cnt);
}

/* polygon point count of each pair (a[i], b[i]), i < n: the reference's box_overlap needs cnt <= 16 */
void oracle_overlap_points(const float *a, const float *b, int n, int32_t *count)
{
    for (int i = 0; i < n; ++i) box_overlap_count(a + (size_t)i * 5, b + (size_t)i * 5, &count[i]);
}

float oracle_iou_bev(const float *a, const float *b)
{
    float sa = (a[2] - a[0]) * (a[3] - a[1]);
    float sb = (b[2] - b[0]) * (b[3] - b[1]);
    float so = oracle_box_overlap(a, b);
    return so / fmaxf(sa + sb - so, kEps);
}

/* Suppression bitmask in the reference layout: mask[i * col_blocks + cb], bit j
 * set when iou(i, cb*64 + j) > thr.  As in the reference kernel, the diagonal
 * tile only evaluates j > i, and off-diagonal tiles (including the lower
 * triangle) are evaluated in full. */
void oracle_nms_mask(const float *boxes, int n, float thr, uint64_t *mask)
{
    int col_blocks = (n + 63) / 64;
    for (int i = 0; i < n; ++i) {
        int rb = i / 64;
        for (int cb = 0; cb < col_blocks; ++cb) {
            int cs = n - cb * 64 < 64 ? n - cb * 64 : 64;
            int start = (rb == cb) ? (i % 64) + 1 : 0;
            uint64_t t = 0;
            for (int j = start; j < cs; ++j)
                if (oracle_iou_bev(boxes + (size_t)i * 5, boxes + ((size_t)cb * 64 + j) * 5) > thr)
                    t |= 1ULL << j;
            mask[(size_t)i * col_blocks + cb] = t;
        }
    }
}

/* Greedy sweep (iou3d.cpp:100-116).  keep[] receives indices into the (already
 * score-sorted) box list; returns how many. */
int oracle_nms_greedy(const uint64_t *mask, int n, int64_t *keep)
{
    int col_blocks = (n + 63) / 64;
    uint64_t *remv = (uint64_t *)calloc((size_t)col_blocks > 0 ? col_blocks : 1, sizeof(uint64_t));
    int num = 0;
    for (int i = 0; i < n; ++i) {
        int nb = i / 64, ib = i % 64;
        if (!(remv[nb] & (1ULL << ib))) {
            keep[num++] = i;
            const uint64_t *p = mask + (size_t)i * col_blocks;
            for (int j = nb; j < col_blocks; ++j) remv[j] |= p[j];
        }
    }
    free(remv);
    return num;
}

/* boxes [n,5] sorted by score already; returns number kept. */
int oracle_nms_sorted(const float *boxes, int n, float thr, int64_t *keep)
{
    if (n <= 0) return 0;
    int col_blocks = (n + 63) / 64;
    uint64_t *mask = (uint64_t *)malloc((size_t)n * col_blocks * sizeof(uint64_t));
    if (!mask) return -1;
    oracle_nms_mask(boxes, n, thr, mask);
    int num = oracle_nms_greedy(mask, n, keep);
    free(mask);
    return num;
}

/* dense IoU matrix for diagnostics (min |IoU - thr| in the tests) */
void oracle_iou_matrix(const float *boxes, int n, float *out)
{
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j)
            out[(size_t)i * n + j] = oracle_iou_bev(boxes + (size_t)i * 5, boxes + (size_t)j * 5);
}

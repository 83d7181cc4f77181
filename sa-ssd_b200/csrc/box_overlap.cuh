// Rotated BEV overlap area of two boxes (x1, y1, x2, y2, angle): box_overlap of the reference's
// iou3d_kernel.cu, evaluated expression for expression (same fp32 operation order, same libm calls, same contraction
// opportunities), so that the area is bit-identical to the reference kernel's.  Shared by the NMS (nms.cu) and the
// rotated-3D-IoU target assignment (targets.cu).
#pragma once
#include <cuda_runtime.h>

namespace {

constexpr float kEps = 1e-8f;

struct P2 { float x, y; };

__device__ __forceinline__ float cross_o(const P2& p1, const P2& p2, const P2& p0) {
    return (p1.x - p0.x) * (p2.y - p0.y) - (p2.x - p0.x) * (p1.y - p0.y);
}

__device__ __forceinline__ float cross_v(const P2& a, const P2& b) { return a.x * b.y - a.y * b.x; }

__device__ __forceinline__ bool spans_overlap(const P2& p1, const P2& p2, const P2& q1, const P2& q2) {
    return fminf(p1.x, p2.x) <= fmaxf(q1.x, q2.x) && fminf(q1.x, q2.x) <= fmaxf(p1.x, p2.x) &&
           fminf(p1.y, p2.y) <= fmaxf(q1.y, q2.y) && fminf(q1.y, q2.y) <= fmaxf(p1.y, p2.y);
}

// is p inside the rotated rectangle `box` = (x1,y1,x2,y2,angle), margin 1e-5
__device__ __forceinline__ bool point_in_box(const float* box, const P2& p) {
    const float MARGIN = 1e-5f;
    float center_x = (box[0] + box[2]) / 2;
    float center_y = (box[1] + box[3]) / 2;
    float angle_cos = cosf(-box[4]), angle_sin = sinf(-box[4]);
    float rot_x = (p.x - center_x) * angle_cos + (p.y - center_y) * angle_sin + center_x;
    float rot_y = -(p.x - center_x) * angle_sin + (p.y - center_y) * angle_cos + center_y;
    return (rot_x > box[0] - MARGIN && rot_x < box[2] + MARGIN && rot_y > box[1] - MARGIN && rot_y < box[3] + MARGIN);
}

__device__ __forceinline__ bool edge_hit(const P2& p1, const P2& p0, const P2& q1, const P2& q0, P2& ans) {
    if (!spans_overlap(p0, p1, q0, q1)) return false;
    float s1 = cross_o(q0, p1, p0);
    float s2 = cross_o(p1, q1, p0);
    float s3 = cross_o(p0, q1, q0);
    float s4 = cross_o(q1, p1, q0);
    if (!(s1 * s2 > 0 && s3 * s4 > 0)) return false;
    float s5 = cross_o(q1, p1, p0);
    if (fabsf(s5 - s1) > kEps) {
        ans.x = (s5 * q0.x - s1 * q1.x) / (s5 - s1);
        ans.y = (s5 * q0.y - s1 * q1.y) / (s5 - s1);
    } else {
        float a0 = p0.y - p1.y, b0 = p1.x - p0.x, c0 = p0.x * p1.y - p1.x * p0.y;
        float a1 = q0.y - q1.y, b1 = q1.x - q0.x, c1 = q0.x * q1.y - q1.x * q0.y;
        float D = a0 * b1 - a1 * b0;
        ans.x = (b0 * c1 - b1 * c0) / D;
        ans.y = (a1 * c0 - a0 * c1) / D;
    }
    return true;
}

__device__ __forceinline__ void spin(const P2& center, float angle_cos, float angle_sin, P2& p) {
    float new_x = (p.x - center.x) * angle_cos + (p.y - center.y) * angle_sin + center.x;
    float new_y = -(p.x - center.x) * angle_sin + (p.y - center.y) * angle_cos + center.y;
    p.x = new_x;
    p.y = new_y;
}

__device__ float rotated_overlap(const float* box_a, const float* box_b) {
    float a_x1 = box_a[0], a_y1 = box_a[1], a_x2 = box_a[2], a_y2 = box_a[3], a_angle = box_a[4];
    float b_x1 = box_b[0], b_y1 = box_b[1], b_x2 = box_b[2], b_y2 = box_b[3], b_angle = box_b[4];
    P2 center_a{(a_x1 + a_x2) / 2, (a_y1 + a_y2) / 2};
    P2 center_b{(b_x1 + b_x2) / 2, (b_y1 + b_y2) / 2};
    P2 ca[5] = {{a_x1, a_y1}, {a_x2, a_y1}, {a_x2, a_y2}, {a_x1, a_y2}, {0.f, 0.f}};
    P2 cb[5] = {{b_x1, b_y1}, {b_x2, b_y1}, {b_x2, b_y2}, {b_x1, b_y2}, {0.f, 0.f}};
    float a_angle_cos = cosf(a_angle), a_angle_sin = sinf(a_angle);
    float b_angle_cos = cosf(b_angle), b_angle_sin = sinf(b_angle);
    for (int k = 0; k < 4; k++) {
        spin(center_a, a_angle_cos, a_angle_sin, ca[k]);
        spin(center_b, b_angle_cos, b_angle_sin, cb[k]);
    }
    ca[4] = ca[0];
    cb[4] = cb[0];

    P2 poly[16];
    P2 pc{0.f, 0.f};
    int cnt = 0;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++)
            if (edge_hit(ca[i + 1], ca[i], cb[j + 1], cb[j], poly[cnt])) {
                pc.x = pc.x + poly[cnt].x;
                pc.y = pc.y + poly[cnt].y;
                cnt++;
            }
    for (int k = 0; k < 4; k++) {
        if (point_in_box(box_a, cb[k])) {
            pc.x = pc.x + cb[k].x;
            pc.y = pc.y + cb[k].y;
            poly[cnt] = cb[k];
            cnt++;
        }
        if (point_in_box(box_b, ca[k])) {
            pc.x = pc.x + ca[k].x;
            pc.y = pc.y + ca[k].y;
            poly[cnt] = ca[k];
            cnt++;
        }
    }
    pc.x /= cnt;
    pc.y /= cnt;
    // bubble sort by polar angle about the centroid (same comparison sequence as the reference,
    // so ties and near-ties order identically)
    for (int j = 0; j < cnt - 1; j++)
        for (int i = 0; i < cnt - j - 1; i++)
            if (atan2f(poly[i].y - pc.y, poly[i].x - pc.x) > atan2f(poly[i + 1].y - pc.y, poly[i + 1].x - pc.x)) {
                P2 t = poly[i];
                poly[i] = poly[i + 1];
                poly[i + 1] = t;
            }
    float area = 0;
    for (int k = 0; k < cnt - 1; k++) {
        P2 u{poly[k].x - poly[0].x, poly[k].y - poly[0].y};
        P2 v{poly[k + 1].x - poly[0].x, poly[k + 1].y - poly[0].y};
        area += cross_v(u, v);
    }
    return fabsf(area) / 2.0f;
}

}  // namespace

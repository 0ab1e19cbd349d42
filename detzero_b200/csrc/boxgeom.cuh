// boxgeom.cuh -- rotated-BEV box geometry shared by the NMS / IoU kernels (head.cu), the tracker / crop kernels (track.cu) and the
// weighted box fusion of test-time augmentation (tta.cu); the point-in-box test is shared by the object crop (track.cu) and the
// refiner input builder (refine_data.cu).
// Same polygon-clip algorithm as the reference (utils/detzero_utils/ops/iou3d_nms/src/iou3d_nms_kernel.cu:42-335): the keep set of
// the NMS and the tracker's association matrix depend on its 1e-2 in-box margin and atan2 ordering, so it is re-expressed, not changed.
#pragma once
#include <cuda_runtime.h>

struct P2 { float x, y; };

// Both products are rounded before the difference (no FMA contraction), so cross_o(a, b, o) == -cross_o(b, a, o) exactly.
// seg_hit relies on it: s1 * s2 > 0 must imply that s1 and s5 = -s2 have opposite signs, which keeps the crossing point between
// q0 and q1.  With a contracted product the two sides of two collinear edges (abutting boxes, boxes turned by k*pi/2) come out
// as unrelated rounding noise, and the crossing point can land metres outside both boxes.
__device__ __forceinline__ float cross_o(P2 a, P2 b, P2 o) {
    return __fsub_rn(__fmul_rn(a.x - o.x, b.y - o.y), __fmul_rn(b.x - o.x, a.y - o.y));
}

__device__ __forceinline__ bool seg_hit(P2 p1, P2 p0, P2 q1, P2 q0, P2& out) {
    bool bb = fminf(p0.x, p1.x) <= fmaxf(q0.x, q1.x) && fminf(q0.x, q1.x) <= fmaxf(p0.x, p1.x) &&
              fminf(p0.y, p1.y) <= fmaxf(q0.y, q1.y) && fminf(q0.y, q1.y) <= fmaxf(p0.y, p1.y);
    if (!bb) return false;
    float s1 = cross_o(q0, p1, p0), s2 = cross_o(p1, q1, p0);
    float s3 = cross_o(p0, q1, q0), s4 = cross_o(q1, p1, q0);
    if (!(s1 * s2 > 0.f && s3 * s4 > 0.f)) return false;
    float s5 = cross_o(q1, p1, p0);
    if (fabsf(s5 - s1) > 1e-8f) {
        out.x = (s5 * q0.x - s1 * q1.x) / (s5 - s1);
        out.y = (s5 * q0.y - s1 * q1.y) / (s5 - s1);
    } else {
        float a0 = p0.y - p1.y, b0 = p1.x - p0.x, c0 = p0.x * p1.y - p1.x * p0.y;
        float a1 = q0.y - q1.y, b1 = q1.x - q0.x, c1 = q0.x * q1.y - q1.x * q0.y;
        float D = a0 * b1 - a1 * b0;
        out.x = (b0 * c1 - b1 * c0) / D;
        out.y = (a1 * c0 - a0 * c1) / D;
    }
    return true;
}

__device__ __forceinline__ bool inside_box(const float* box, P2 p) {
    float cs = cosf(-box[6]), sn = sinf(-box[6]);
    float dx = p.x - box[0], dy = p.y - box[1];
    float rx = dx * cs + dy * (-sn), ry = dx * sn + dy * cs;
    return fabsf(rx) < box[3] / 2 + 1e-2f && fabsf(ry) < box[4] / 2 + 1e-2f;
}

__device__ __forceinline__ void box_corners(const float* box, P2* c) {
    float hx = box[3] / 2, hy = box[4] / 2, cs = cosf(box[6]), sn = sinf(box[6]);
    const float sx[4] = {-1.f, 1.f, 1.f, -1.f}, sy[4] = {-1.f, -1.f, 1.f, 1.f};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        float px = box[0] + sx[k] * hx, py = box[1] + sy[k] * hy;       // axis-aligned corner, then rotate about centre
        c[k].x = (px - box[0]) * cs + (py - box[1]) * (-sn) + box[0];
        c[k].y = (px - box[0]) * sn + (py - box[1]) * cs + box[1];
    }
    c[4] = c[0];
}

static __device__ float bev_overlap(const float* a, const float* b) {
    P2 A[5], Bc[5];
    box_corners(a, A);
    box_corners(b, Bc);
    P2 pts[16];
    float ang[16];
    int cnt = 0;
    float cx = 0.f, cy = 0.f;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            P2 h;
            if (seg_hit(A[i + 1], A[i], Bc[j + 1], Bc[j], h)) { pts[cnt++] = h; cx += h.x; cy += h.y; }
        }
    for (int k = 0; k < 4; ++k) {
        if (inside_box(a, Bc[k])) { pts[cnt++] = Bc[k]; cx += Bc[k].x; cy += Bc[k].y; }
        if (inside_box(b, A[k])) { pts[cnt++] = A[k]; cx += A[k].x; cy += A[k].y; }
    }
    if (cnt < 3) return 0.f;
    cx /= cnt; cy /= cnt;
    for (int i = 0; i < cnt; ++i) ang[i] = atan2f(pts[i].y - cy, pts[i].x - cx);
    for (int i = 1; i < cnt; ++i) {              // stable insertion sort, ascending angle
        P2 p = pts[i]; float t = ang[i];
        int j = i - 1;
        while (j >= 0 && ang[j] > t) { pts[j + 1] = pts[j]; ang[j + 1] = ang[j]; --j; }
        pts[j + 1] = p; ang[j + 1] = t;
    }
    float area = 0.f;
    for (int k = 0; k < cnt - 1; ++k)
        area += (pts[k].x - pts[0].x) * (pts[k + 1].y - pts[0].y) - (pts[k].y - pts[0].y) * (pts[k + 1].x - pts[0].x);
    return fabsf(area) / 2.f;
}

// centre distance beyond the sum of half-diagonals plus 0.05 m: the BEV overlap of the two boxes is exactly 0 (no corner lies
// within the 1e-2 in-box margin, no edges cross); the tracker and the ground-truth scoring skip such pairs before bev_overlap
__device__ __forceinline__ bool far_pair(const float* a, const float* b) {
    const float dx = a[0] - b[0], dy = a[1] - b[1];
    const float r = 0.5f * (sqrtf(a[3] * a[3] + a[4] * a[4]) + sqrtf(b[3] * b[3] + b[4] * b[4])) + 0.05f;
    return dx * dx + dy * dy > r * r;
}

__device__ __forceinline__ float bev_iou(const float* a, const float* b) {
    float sa = a[3] * a[4], sb = b[3] * b[4];
    float so = bev_overlap(a, b);
    return so / fmaxf(sa + sb - so, 1e-8f);
}

// 3-D IoU of boxes_iou3d_gpu (iou3d_nms_utils.py:85-105): BEV overlap area times the z overlap, over the union volume
__device__ __forceinline__ float iou3d(const float* a, const float* b) {
    const float a_max = a[2] + a[5] / 2, a_min = a[2] - a[5] / 2, b_max = b[2] + b[5] / 2, b_min = b[2] - b[5] / 2;
    const float oh = fmaxf(fminf(a_max, b_max) - fmaxf(a_min, b_min), 0.f);
    const float o3 = bev_overlap(a, b) * oh;
    return o3 / fmaxf(a[3] * a[4] * a[5] + b[3] * b[4] * b[5] - o3, 1e-6f);
}

// roiaware_pool3d_kernel.cu:16-36 (check_pt_in_box3d, GPU margin 1e-5; the z test has no margin)
__device__ __forceinline__ bool pt_in_box3d(float x, float y, float z, const float* b) {
    if (fabsf(z - b[2]) > b[5] / 2.0f) return false;
    const float sx = x - b[0], sy = y - b[1];
    const float cosa = cosf(-b[6]), sina = sinf(-b[6]);
    const float lx = sx * cosa + sy * (-sina), ly = sx * sina + sy * cosa;
    return (fabsf(lx) < b[3] / 2.0f + 1e-5f) & (fabsf(ly) < b[4] / 2.0f + 1e-5f);
}

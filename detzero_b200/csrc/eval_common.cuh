// eval_common.cuh -- device pieces shared by the scorings against ground truth: det_eval.cu (Waymo AP / APH), track_gt.cu (tracks
// against ground truth) and track_eval.cu (Waymo MOTA / MOTP); yawf also by the tracker (tracker.cu).
#pragma once
#include <cuda_runtime.h>

namespace {

// score cutoff k of the Waymo configs (0..100): float32(k * 0.01), the last 1.0; a prediction is active at k when score >= it
__device__ __forceinline__ float score_cutoff(int k) { return k < 100 ? __double2float_rn(__dmul_rn((double)k, 0.01)) : 1.f; }

// RANGE breakdown bin of a box centre: [0, 30) / [30, 50) / [50, +inf) of the float32 sqrt(x^2 + y^2), no FMA contraction
__device__ __forceinline__ int range_bin(float x, float y) {
    const float r = __fsqrt_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
    return r < 30.f ? 0 : (r < 50.f ? 1 : 2);
}

__device__ __forceinline__ float yawf(float y) {                      // transform_utils.yaw_filter, ndarray branch, float32
    const float pi2 = 6.283185307179586f, pi = 3.141592653589793f;
    if (fabsf(y) >= pi2) y = y - floorf(y / pi2) * pi2;
    if (y > pi) y -= pi2;
    if (y <= -pi) y += pi2;
    return y;
}

// a track entry's world box b (9 doubles) back to the lidar frame of pose Pm (4 x 4 lidar -> world, row-major) as
// tracklets_to_frames / transform_boxes3d(inverse=True) do it: the box cast to float32, the inverse pose rounded to float32
// (get_inverse_transform_mat), the centre product in float64 rounded to float32, the heading through the float32 yaw_filter -> l[7]
__device__ __forceinline__ void entry_to_lidar(const double* b, const double* Pm, float* l) {
    float inv[12];
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) inv[r * 4 + c] = (float)Pm[c * 4 + r];
        double t = __dmul_rn(Pm[r], Pm[3]);
        t = __dadd_rn(t, __dmul_rn(Pm[4 + r], Pm[7]));
        t = __dadd_rn(t, __dmul_rn(Pm[8 + r], Pm[11]));
        inv[r * 4 + 3] = (float)(-t);
    }
    const float x = (float)b[0], y = (float)b[1], z = (float)b[2];
    for (int r = 0; r < 3; ++r) {
        double c = __dmul_rn((double)x, (double)inv[r * 4]);
        c = __dadd_rn(c, __dmul_rn((double)y, (double)inv[r * 4 + 1]));
        c = __dadd_rn(c, __dmul_rn((double)z, (double)inv[r * 4 + 2]));
        l[r] = (float)__dadd_rn(c, (double)inv[r * 4 + 3]);
    }
    l[3] = (float)b[3]; l[4] = (float)b[4]; l[5] = (float)b[5];
    l[6] = yawf(__fadd_rn((float)b[6], (float)atan2((double)inv[4], (double)inv[0])));
}

}  // namespace

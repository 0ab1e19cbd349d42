// refine_frame.cuh -- the init-box frame of a track (refining/detzero_refine/utils/data_utils.py:72-106, init_coords_transform),
// shared by the refiner input builder (refine_data.cu: pos_trajectory) and the ground-truth targets (refine_gt.cu:
// gt_pos_trajectory), so that a track's boxes and its ground truth go through the same float64 arithmetic.
#pragma once
#include <cuda_runtime.h>

// data_utils.limit_heading_range: into [-pi, pi)
__device__ __forceinline__ double wrap_pi(double a) {
    const double PI = 3.14159265358979323846;
    while (a >= PI) a -= 2 * PI;
    while (a < -PI) a += 2 * PI;
    return a;
}

struct InitFrame { double yaw, c, s; };

// the frame of the init box bi (x, y, z, dx, dy, dz, heading): its heading wrapped, and the rotation by -heading
__device__ __forceinline__ InitFrame init_frame(const double* bi) {
    InitFrame fr;
    fr.yaw = wrap_pi(bi[6]);
    fr.c = cos(fr.yaw);
    fr.s = sin(fr.yaw);
    return fr;
}

// the world box bw in the frame of the init box bi
__device__ __forceinline__ void to_init_frame(const InitFrame& fr, const double* bi, const double* bw, double loc[7]) {
    const double dx = bw[0] - bi[0], dy = bw[1] - bi[1], dz = bw[2] - bi[2];
    loc[0] = fr.c * dx + fr.s * dy;
    loc[1] = -fr.s * dx + fr.c * dy;
    loc[2] = dz;
    loc[3] = bw[3]; loc[4] = bw[4]; loc[5] = bw[5];
    loc[6] = wrap_pi(wrap_pi(bw[6]) - fr.yaw);
}

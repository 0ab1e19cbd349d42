// assign.cuh -- the exact rectangular assignment shared by the tracker's association (tracker.cu) and the ground-truth trajectory
// assignment (track_gt.cu): union-find labels of the valid-edge graph, the Hungarian method with potentials on one thread, and the
// same method with every column loop spread over the block.  Both solvers use the same arithmetic and take the first minimum of an
// ascending column scan, so a component gives the same assignment whichever of them solves it.
#pragma once
#include <float.h>
#include <limits.h>
#include <cuda_runtime.h>

namespace {

__device__ __forceinline__ int uf_find(volatile int* lab, int x) {
    int p = lab[x];
    while (p != x) { x = p; p = lab[x]; }
    return x;
}

// exact rectangular assignment (Hungarian with potentials, rows <= cols), a row-major n x m; p[j] = row (1-based) of column j
__device__ void hungarian(const double* a, int n, int m, double* u, double* v, double* minv, int* p, int* way, unsigned char* used) {
    for (int j = 0; j <= m; ++j) { v[j] = 0.; p[j] = 0; way[j] = 0; }
    for (int i = 0; i <= n; ++i) u[i] = 0.;
    for (int i = 1; i <= n; ++i) {
        p[0] = i;
        int j0 = 0;
        for (int j = 0; j <= m; ++j) { minv[j] = DBL_MAX; used[j] = 0; }
        do {
            used[j0] = 1;
            const int i0 = p[j0];
            double delta = DBL_MAX;
            int j1 = 0;
            for (int j = 1; j <= m; ++j)
                if (!used[j]) {
                    const double cur = a[(size_t)(i0 - 1) * m + (j - 1)] - u[i0] - v[j];
                    if (cur < minv[j]) { minv[j] = cur; way[j] = j0; }
                    if (minv[j] < delta) { delta = minv[j]; j1 = j; }
                }
            for (int j = 0; j <= m; ++j)
                if (used[j]) { u[p[j]] += delta; v[j] -= delta; } else minv[j] -= delta;
            j0 = j1;
        } while (p[j0] != 0);
        do { const int j1 = way[j0]; p[j0] = p[j1]; j0 = j1; } while (j0);
    }
}

// block-wide reduction scratch of hungarian_block for a block of NT threads (NT a multiple of 32)
template <int NT>
struct HungShared {
    double wval[NT / 32], hdelta;   // per-warp minima; the step's delta
    int widx[NT / 32], hj1;         // their columns; the step's column
};

// (value, index) minimum over the block, the smaller index on a tie -> sh.hdelta, sh.hj1 (the first minimum of an ascending scan)
template <int NT>
__device__ void block_argmin(double val, int idx, HungShared<NT>& sh) {
    constexpr int NW = NT / 32;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int off = 16; off; off >>= 1) {
        const double ov = __shfl_down_sync(0xffffffffu, val, off);
        const int oi = __shfl_down_sync(0xffffffffu, idx, off);
        if (ov < val || (ov == val && oi < idx)) { val = ov; idx = oi; }
    }
    if (lane == 0) { sh.wval[w] = val; sh.widx[w] = idx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double bv = sh.wval[0];
        int bi = sh.widx[0];
        for (int k = 1; k < NW; ++k)
            if (sh.wval[k] < bv || (sh.wval[k] == bv && sh.widx[k] < bi)) { bv = sh.wval[k]; bi = sh.widx[k]; }
        sh.hdelta = bv; sh.hj1 = bi;
    }
    __syncthreads();
}

// hungarian() with every column loop spread over the block: the same arithmetic on every element and the same (first) minimum,
// so the result is that of the one-thread solver.  Each augmentation step costs two block reductions.
template <int NT>
__device__ void hungarian_block(const double* a, int n, int m, double* u, double* v, double* minv, int* p, int* way,
                                unsigned char* used, HungShared<NT>& sh) {
    for (int j = threadIdx.x; j <= m; j += NT) { v[j] = 0.; p[j] = 0; way[j] = 0; }
    for (int i = threadIdx.x; i <= n; i += NT) u[i] = 0.;
    __syncthreads();
    for (int i = 1; i <= n; ++i) {
        for (int j = threadIdx.x; j <= m; j += NT) { minv[j] = DBL_MAX; used[j] = 0; }
        if (threadIdx.x == 0) p[0] = i;
        __syncthreads();
        int j0 = 0;
        while (true) {
            if (threadIdx.x == 0) used[j0] = 1;
            __syncthreads();
            const int i0 = p[j0];
            const double ui0 = u[i0];
            double best = DBL_MAX;
            int bj = INT_MAX;
            for (int j = 1 + threadIdx.x; j <= m; j += NT)
                if (!used[j]) {
                    const double cur = a[(size_t)(i0 - 1) * m + (j - 1)] - ui0 - v[j];
                    if (cur < minv[j]) { minv[j] = cur; way[j] = j0; }
                    if (minv[j] < best) { best = minv[j]; bj = j; }
                }
            block_argmin<NT>(best, bj, sh);
            const double delta = sh.hdelta;
            const int j1 = sh.hj1;
            for (int j = threadIdx.x; j <= m; j += NT)
                if (used[j]) { u[p[j]] += delta; v[j] -= delta; } else minv[j] -= delta;
            __syncthreads();
            j0 = j1;
            if (p[j0] == 0) break;
        }
        if (threadIdx.x == 0)
            do { const int j1 = way[j0]; p[j0] = p[j1]; j0 = j1; } while (j0);
        __syncthreads();
    }
}

}  // namespace

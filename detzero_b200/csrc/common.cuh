// common.cuh -- shared helpers for libdetzero_b200 (sm_90a).
#pragma once
#include <stdlib.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/detzero_b200.h"

#define DZ_NUM_SMS 132

void dz_set_error(const char* fmt, ...);

#define DZ_CHECK_ARG(cond)                                                            \
    do { if (!(cond)) { dz_set_error("%s:%d: bad argument: %s", __FILE__, __LINE__, #cond); return DZ_ERR_ARG; } } while (0)

#define DZ_CUDA(call)                                                                 \
    do { cudaError_t e__ = (call); if (e__ != cudaSuccess) {                          \
        dz_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); return DZ_ERR_CUDA; } } while (0)

#define DZ_LAUNCH_CHECK()                                                             \
    do { cudaError_t e__ = cudaGetLastError(); if (e__ != cudaSuccess) {              \
        dz_set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(e__)); return DZ_ERR_CUDA; } } while (0)

static inline size_t dz_align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int dz_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// carve a workspace
struct DzWs {
    char* p; size_t left;
    DzWs(void* ws, size_t bytes) : p((char*)ws), left(bytes) {}
    template <typename T> T* take(size_t n) {
        size_t b = dz_align_up(n * sizeof(T), 256);
        if (b > left) return nullptr;
        T* r = (T*)p; p += b; left -= b; return r;
    }
};

// ---- grid index lookup (device) ----------------------------------------------------------------------------
struct GridIndex {
    const uint32_t* bitmap;
    const uint32_t* prefix;
    const int32_t* perm;      // may be null (identity)
    int B, D, H, W;
    long long cells_pad;      // round_up(D*H*W, 32)
    int rows;                 // capacity of the indexed tensor: with an identity perm, a rank >= rows has no row
};

static inline long long dz_cells_pad(int D, int H, int W) {
    long long c = (long long)D * H * W;
    return (c + 31) / 32 * 32;
}

__device__ __forceinline__ int grid_lookup(const GridIndex& g, int b, int z, int y, int x) {
    if ((unsigned)z >= (unsigned)g.D || (unsigned)y >= (unsigned)g.H || (unsigned)x >= (unsigned)g.W) return -1;
    long long cell = (long long)b * g.cells_pad + ((long long)z * g.H + y) * g.W + x;
    size_t w = (size_t)(cell >> 5);
    uint32_t bit = (uint32_t)cell & 31u;
    uint32_t word = __ldg(g.bitmap + w);
    if (!((word >> bit) & 1u)) return -1;
    int rank = (int)(__ldg(g.prefix + w) + __popc(word & ((1u << bit) - 1u)));
    // a level whose count overflowed its capacity still has every site in its bitmap; those beyond the capacity have no row
    // (the overflow is reported and the frame re-run), so they must not reach a neighbour table
    return g.perm ? __ldg(g.perm + rank) : (rank < g.rows ? rank : -1);
}

__device__ __forceinline__ int warp_inclusive_scan(int v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// block-wide exclusive scan of one int per thread (blockDim.x <= 1024, multiple of 32). returns the exclusive
// prefix; *total gets the block sum (valid in all threads).  Safe to call repeatedly.
__device__ __forceinline__ int block_exclusive_scan(int v, int* total) {
    __shared__ int ws_scan[33];
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int inc = warp_inclusive_scan(v, lane);
    if (lane == 31) ws_scan[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        int nw = blockDim.x >> 5;
        int s = lane < nw ? ws_scan[lane] : 0;
        int si = warp_inclusive_scan(s, lane);
        ws_scan[lane] = si - s;
        if (lane == 31) ws_scan[32] = si;
    }
    __syncthreads();
    *total = ws_scan[32];
    int r = ws_scan[wid] + inc - v;
    __syncthreads();
    return r;
}

// ordered block-wide compaction: emit(i, pos) for the items i < n with pred(i) true, pos counting them in index order; returns
// the count.  Every emit is visible to the whole block on return.
template <class Pred, class Emit>
__device__ int block_compact(int n, Pred pred, Emit emit) {
    int total = 0;
    for (int base = 0; base < n; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const int q = i < n && pred(i);
        int sum;
        const int pos = block_exclusive_scan(q, &sum);
        if (q) emit(i, total + pos);
        total += sum;
    }
    __syncthreads();
    return total;
}

// a workspace carved in 256-byte aligned pieces, the same list on the host and the device: from a null base it only adds up the
// bytes, which is how the *_ws_bytes entry points size it
struct DzCarve {
    char* base;
    size_t bytes = 0;
    __host__ __device__ explicit DzCarve(char* b) : base(b) {}
    template <typename T> __host__ __device__ T* take(size_t n) {
        T* r = (T*)(base + bytes);
        bytes += (n * sizeof(T) + 255) / 256 * 256;
        return r;
    }
};

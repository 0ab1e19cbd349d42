// assign.cuh -- the exact assignment by connected components of a valid-edge graph, shared by the tracker's association
// (tracker.cu), the ground-truth trajectory assignment (track_gt.cu) and the Waymo scorings (det_eval.cu, track_eval.cu):
//
//   uf_label / group_edges   min-hooking union-find labels of the edge graph, then the edges grouped by component root
//   sort_edges               a small component's edges in (row, column) order on one thread
//   solve_dense(_block)      one component as a dense cost matrix (rows the smaller side) solved by the Hungarian method with
//                            potentials, on one thread (hungarian) or with every column loop spread over the block (hungarian_block)
//
// Both solvers use the same arithmetic and take the first minimum of an ascending column scan, so a cost matrix gives the same
// assignment whichever of them solves it; the order of the local rows and columns is the caller's and decides exact ties.  Each
// caller keeps its edge list, its component loops and its cost convention.
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

// min-hooking union-find over the edges e < ne joining node row(e) to node col(e): lab (lab[v] = v, preset by the caller) ends
// with every node's component rooted at its smallest node.  changed: a shared flag of the block.
template <int NT, class Row, class Col>
__device__ void uf_label(int* lab, int ne, Row row, Col col, int& changed) {
    volatile int* vl = lab;
    while (ne) {
        if (threadIdx.x == 0) changed = 0;
        __syncthreads();
        for (int e = threadIdx.x; e < ne; e += NT) {
            const int a = uf_find(vl, row(e)), b = uf_find(vl, col(e));
            if (a != b) { atomicMin(&lab[max(a, b)], min(a, b)); changed = 1; }
        }
        __syncthreads();
        const int ch = changed;
        __syncthreads();
        if (!ch) break;
    }
}

// the edges (er, ec, ew)[e < ne] grouped by component into (sr, sc, sw), where every root is a row node r < nrows: rcnt (zeroed
// for the rows by the caller) ends as each root's end offset, so a component is [rcnt[root - 1], rcnt[root]) (from 0 for row 0)
template <int NT>
__device__ void group_edges(int* lab, int ne, int nrows, int* rcnt, const int* er, const int* ec, const float* ew, int* sr, int* sc,
                            float* sw) {
    for (int e = threadIdx.x; e < ne; e += NT) atomicAdd(&rcnt[uf_find(lab, er[e])], 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int r = 0; r < nrows; ++r) { const int c = rcnt[r]; rcnt[r] = run; run += c; }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < ne; e += NT) {
        const int pos = atomicAdd(&rcnt[uf_find(lab, er[e])], 1);
        sr[pos] = er[e]; sc[pos] = ec[e]; sw[pos] = ew[e];
    }
    __syncthreads();
}

// a small component's m edges sorted by (row, column) on one thread: a deterministic component whatever the grouping order
__device__ void sort_edges(int* er, int* ec, float* ew, int m) {
    for (int i = 1; i < m; ++i) {
        const int r = er[i], c = ec[i];
        const float a = ew[i];
        int j = i - 1;
        while (j >= 0 && (er[j] > r || (er[j] == r && ec[j] > c))) { er[j + 1] = er[j]; ec[j + 1] = ec[j]; ew[j + 1] = ew[j]; --j; }
        er[j + 1] = r; ec[j + 1] = c; ew[j + 1] = a;
    }
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

// doubles of scratch a component of nr rows and nc columns takes: the (smaller side) x (larger side) cost matrix, then the
// Hungarian's u, v, minv, p, way and used (hungarian_carve)
__host__ __device__ constexpr size_t hungarian_scratch(int nr, int nc) {
    const size_t hn = nr < nc ? nr : nc, hm = nr < nc ? nc : nr;
    return hn * hm + (hn + 1) + 2 * (hm + 1) + (hm + 1) + (hm + 1) / 8 + 2;
}

struct HungArrays {
    double *u, *v, *minv;
    int *p, *way;
    unsigned char* used;
};

// the Hungarian's arrays after an hn x hm cost matrix A
__device__ __forceinline__ HungArrays hungarian_carve(double* A, int hn, int hm) {
    HungArrays h;
    h.u = A + (size_t)hn * hm;
    h.v = h.u + hn + 1;
    h.minv = h.v + hm + 1;
    h.p = (int*)(h.minv + hm + 1);
    h.way = h.p + hm + 1;
    h.used = (unsigned char*)(h.way + hm + 1);
    return h;
}

// one component of nr local rows and nc local columns on one thread.  edge(i, r, c, cost) gives the i-th of m edges as (local row,
// local column, cost), or false to leave it out; every other entry of the matrix is pad.  The rows of the matrix are the smaller
// side (the transpose when nr > nc).  match(r, c) gets every assigned (local row, local column) whose cost is below bound.  scr:
// hungarian_scratch(nr, nc) doubles.
template <class Edge, class Match>
__device__ void solve_dense(int nr, int nc, int m, Edge edge, double pad, double bound, double* scr, Match match) {
    const bool tr = nr > nc;
    const int hn = tr ? nc : nr, hm = tr ? nr : nc;
    for (int k = 0; k < hn * hm; ++k) scr[k] = pad;
    for (int i = 0; i < m; ++i) {
        int r, c;
        double cost;
        if (edge(i, r, c, cost)) scr[tr ? (size_t)c * hm + r : (size_t)r * hm + c] = cost;
    }
    const HungArrays h = hungarian_carve(scr, hn, hm);
    hungarian(scr, hn, hm, h.u, h.v, h.minv, h.p, h.way, h.used);
    for (int j = 1; j <= hm; ++j) {
        if (!h.p[j]) continue;
        const int hi = h.p[j] - 1, hj = j - 1;
        if (!(scr[(size_t)hi * hm + hj] < bound)) continue;
        if (tr) match(hj, hi); else match(hi, hj);
    }
}

// solve_dense with the whole block of NT threads: edge is called for i < m spread over the block, and match for the assigned pairs
// spread over the block; the caller synchronises before it reads what match wrote
template <int NT, class Edge, class Match>
__device__ void solve_dense_block(int nr, int nc, int m, Edge edge, double pad, double bound, double* scr, HungShared<NT>& sh,
                                  Match match) {
    const bool tr = nr > nc;
    const int hn = tr ? nc : nr, hm = tr ? nr : nc;
    for (size_t k = threadIdx.x; k < (size_t)hn * hm; k += NT) scr[k] = pad;
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += NT) {
        int r, c;
        double cost;
        if (edge(i, r, c, cost)) scr[tr ? (size_t)c * hm + r : (size_t)r * hm + c] = cost;
    }
    __syncthreads();
    const HungArrays h = hungarian_carve(scr, hn, hm);
    hungarian_block<NT>(scr, hn, hm, h.u, h.v, h.minv, h.p, h.way, h.used, sh);
    for (int j = 1 + threadIdx.x; j <= hm; j += NT) {
        if (!h.p[j]) continue;
        const int hi = h.p[j] - 1, hj = j - 1;
        if (!(scr[(size_t)hi * hm + hj] < bound)) continue;
        if (tr) match(hj, hi); else match(hi, hj);
    }
}

}  // namespace

// pointmlp_train.cu -- train-mode chains of [Conv1d(k=1) | BatchNorm(batch statistics) | ReLU] layers over token-major rows,
// storing each layer's pre-BatchNorm output z once; normalise + ReLU are applied to an operand as it is loaded.
//
// Replaces, for the GRM (refining/detzero_refine/models/modules/geometry_transformer.py:118-133 in training: memory_encoder ->
// max -> memory_mlp on cat([y2, g]), query_encoder -> max) the conv, BatchNorm and ReLU outputs autograd writes per layer and the
// separate BatchNorm passes over them:
//   dz_pm_fwd       z = act_in(x) W^T (+ a per-group shift), act(z) = ReLU(a z + b): writes z, per-tile column sums of z and z^2
//                   and, optionally, per-tile column max / min of z with their lowest row
//   dz_pm_dgrad     dH_low = (sum over up to two layers of dZ_s W_s) * [a_low z_low + b_low > 0], dZ formed on the fly from the
//                   layer's dH, z and BN-backward table; per-tile column sums of dH_low and dH_low * xhat_low
//   dz_pm_wgrad     dW = dZ^T act_in(x), reduced over all rows: per-CTA partials over fixed row ranges, summed in a fixed order
//   dz_pm_dh        dH = dY [a z + b > 0] with its per-tile sums (the layer whose output gradient comes from outside)
//   dz_pm_act       y = ReLU(a z + b)
//   dz_pm_reduce_tiles / dz_pm_group_ext   the per-tile partials reduced over each group of tiles in ascending order
//
// A layer's table is (6, N) floats: a = gamma rstd, b = beta - mean a, mean, rstd, m1 = sum dH / R, m2 = sum dH xhat / R; the BN
// backward is dZ = a (dH - m1 - xhat m2), xhat = (z - mean) rstd.  A pooled gradient (dH non-zero only at one row per group and
// channel) is given as (sel, dsel): the row within the group and the value.
// Tiles: 64 rows x 128 columns per CTA (forward / dgrad, M = rows), 64 output channels x 128 input columns over a range of rows
// (wgrad, M = channels, the rows the reduction).  The reduction is staged 32 floats (one 128-byte swizzle atom) at a time in two
// shared-memory stages: a thread loads four consecutive channels per 16-byte load, with their BN tables once per chunk (once per
// CTA in the wgrad), and stages chunk c + 1 while the asynchronous wgmmas of chunk c run.
// Modes: DZ_F32 = exact fp32 FMA; DZ_TF32 = wgmma m64n128k8 TF32 with operands rounded to nearest.  TF32 wgmma takes K-major
// operands only: the forward and dgrad operands are K-major as stored (x / dZ rows, W rows / W^T rows); the wgrad operands
// reduce over rows and are transposed on their way into shared memory.  The fp32 path reads the same shared-memory tiles and
// accumulates into the same fragment layout, so both modes share every epilogue.
// Determinism: every partial has one owner and is reduced in a fixed order; the same inputs give the same bits.
#include "common.cuh"
#include "tc.cuh"

namespace {

constexpr int TM = 64;            // rows per tile (forward / dgrad) = output channels per tile (wgrad)
constexpr int TN = 128;           // output columns per CTA
constexpr int KC = 32;            // reduction chunk (floats): one 128-byte swizzle atom
constexpr int NTH = 128;          // one warpgroup
constexpr int A_BYTES = TM * KC * 4, B_BYTES = TN * KC * 4;
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int SMEM_BYTES = 2 * STAGE_BYTES + 1024;     // two stages: one is staged while the MMAs read the other
enum { T_A = 0, T_B = 1, T_MU = 2, T_RS = 3, T_M1 = 4, T_M2 = 5 };

// float index of (row r, k) in a K-major tile of 128-byte rows with the 128-byte swizzle (16-byte chunk k/4 ^ r%8)
__device__ __forceinline__ int swz(int r, int k) { return r * 32 + ((((k >> 2) ^ (r & 7)) << 2) | (k & 3)); }

template <int MODE>
__device__ __forceinline__ float opnd(float v) { return MODE == DZ_TF32 ? tc::rna_tf32(v) : v; }

// one layer's dZ source: dZ(row, n) = a[n] (dH(row, n) - m1[n] - (z - mean[n]) rstd[n] m2[n])
struct Seg {
    int N;                  // channels
    const float* dh;        // (R, N) dense dH, or null: pooled
    const int* sel;         // (groups, N) pooled row within the group
    const float* dsel;      // (groups, N) dH at that row
    const float* z;         // (R, N)
    const float* tab;       // (6, N)
    const float* wt;        // dgrad: (Kout, N) = W^T
};

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// a layer's BN-backward table at four consecutive channels
struct Quad { float4 a, mu, rs, m1, m2; };
__device__ __forceinline__ Quad quad(const float* t, int N, int n) {
    return Quad{ld4(t + T_A * N + n), ld4(t + T_MU * N + n), ld4(t + T_RS * N + n), ld4(t + T_M1 * N + n), ld4(t + T_M2 * N + n)};
}
__device__ __forceinline__ float dz1(float dh, float z, float a, float mu, float rs, float m1, float m2) {
    return a * (dh - m1 - ((z - mu) * rs) * m2);
}
// dZ at four consecutive channels n..n+3 of one row; lrow is the row within its group g (pooled dH)
__device__ __forceinline__ float4 dz4(const Seg& s, const Quad& q, long long row, int n, long long g, int lrow) {
    const float4 z = ld4(s.z + row * s.N + n);
    float4 dh;
    if (s.dh) {
        dh = ld4(s.dh + row * s.N + n);
    } else {
        const int4 sel = __ldg(reinterpret_cast<const int4*>(s.sel + g * s.N + n));
        const float4 ds = ld4(s.dsel + g * s.N + n);
        dh = make_float4(sel.x == lrow ? ds.x : 0.f, sel.y == lrow ? ds.y : 0.f, sel.z == lrow ? ds.z : 0.f, sel.w == lrow ? ds.w : 0.f);
    }
    return make_float4(dz1(dh.x, z.x, q.a.x, q.mu.x, q.rs.x, q.m1.x, q.m2.x), dz1(dh.y, z.y, q.a.y, q.mu.y, q.rs.y, q.m1.y, q.m2.y),
                       dz1(dh.z, z.z, q.a.z, q.mu.z, q.rs.z, q.m1.z, q.m2.z), dz1(dh.w, z.w, q.a.w, q.mu.w, q.rs.w, q.m1.w, q.m2.w));
}
// ReLU(a x + b) at four channels
__device__ __forceinline__ float4 act4(float4 v, float4 a, float4 b) {
    return make_float4(fmaxf(fmaf(a.x, v.x, b.x), 0.f), fmaxf(fmaf(a.y, v.y, b.y), 0.f), fmaxf(fmaf(a.z, v.z, b.z), 0.f),
                       fmaxf(fmaf(a.w, v.w, b.w), 0.f));
}
template <int MODE>
__device__ __forceinline__ float4 opnd4(float4 v) { return make_float4(opnd<MODE>(v.x), opnd<MODE>(v.y), opnd<MODE>(v.z), opnd<MODE>(v.w)); }
// four K-consecutive operand values (k % 4 == 0) into a K-major tile: one 16-byte store
__device__ __forceinline__ void st4(float* T, int r, int k, float4 v) { *reinterpret_cast<float4*>(T + swz(r, k)) = v; }

// acc (m64 n128 fragment: acc[4j + 2r + c] is row 16 w + l/4 + 8 r, column 8 j + 2 (l%4) + c) += A (64 x 32) B (128 x 32)^T
// In TF32 the MMAs are only issued here (asynchronous): the caller stages the next chunk meanwhile and then calls mma_wait.
template <int MODE>
__device__ __forceinline__ void mma_chunk(float (&acc)[64], const float* As, const float* Bs) {
    if constexpr (MODE == DZ_TF32) {
        const uint64_t ad = tc::smem_desc_sw128(tc::smem_u32(As)), bd = tc::smem_desc_sw128(tc::smem_u32(Bs));
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) tc::wgmma<TN, tc::K_TF32>(acc, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), 1u);
        tc::wgmma_commit();
    } else {
        const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
        const int r0 = 16 * w + (l >> 2);
#pragma unroll 1
        for (int k = 0; k < KC; k += 4) {
            const float4 a0 = *reinterpret_cast<const float4*>(As + swz(r0, k));
            const float4 a1 = *reinterpret_cast<const float4*>(As + swz(r0 + 8, k));
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const float4 b = *reinterpret_cast<const float4*>(Bs + swz(8 * j + 2 * (l & 3) + c, k));
                    float& d0 = acc[4 * j + c];
                    float& d1 = acc[4 * j + 2 + c];
                    d0 = fmaf(a0.x, b.x, d0); d0 = fmaf(a0.y, b.y, d0); d0 = fmaf(a0.z, b.z, d0); d0 = fmaf(a0.w, b.w, d0);
                    d1 = fmaf(a1.x, b.x, d1); d1 = fmaf(a1.y, b.y, d1); d1 = fmaf(a1.z, b.z, d1); d1 = fmaf(a1.w, b.w, d1);
                }
        }
    }
}

template <int MODE>
__device__ __forceinline__ void mma_wait() {
    if constexpr (MODE == DZ_TF32) tc::wgmma_wait_all();
}

// The chunk loop shared by the three GEMMs: stage(As, Bs, c) fills chunk c; chunk c + 1 is staged while the MMAs of chunk c run.
template <int MODE, class Stage>
__device__ __forceinline__ void gemm_loop(float (&acc)[64], unsigned char* sm, int chunks, Stage stage) {
    auto A = [&](int b) { return reinterpret_cast<float*>(sm + b * STAGE_BYTES); };
    auto B = [&](int b) { return reinterpret_cast<float*>(sm + b * STAGE_BYTES + A_BYTES); };
    if (chunks <= 0) return;
    stage(A(0), B(0), 0);
    if (MODE == DZ_TF32) tc::fence_proxy_async();
    __syncthreads();
    for (int c = 0; c < chunks; ++c) {
        mma_chunk<MODE>(acc, A(c & 1), B(c & 1));
        if (c + 1 < chunks) stage(A((c + 1) & 1), B((c + 1) & 1), c + 1);     // the other stage: its MMAs were waited for
        mma_wait<MODE>();
        if (MODE == DZ_TF32) tc::fence_proxy_async();
        __syncthreads();
    }
}

__device__ __forceinline__ int frow(int r) { return 16 * (threadIdx.x >> 5) + ((threadIdx.x & 31) >> 2) + 8 * r; }
__device__ __forceinline__ int fcol(int j, int c) { return 8 * j + 2 * (threadIdx.x & 3) + c; }

__device__ __forceinline__ unsigned char* smem_base(unsigned char* raw) {
    return reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
}

// per-tile column sums of u(i) and v(i) over the fragment's 64 rows (float64, rows in a fixed order), written to
// ps[0 * ld + col0 + n] and ps[1 * ld + col0 + n].  red: 8 KB of shared memory no thread still reads.
template <class F>
__device__ __forceinline__ void tile_sums(F uv, double* red, double* ps, long long ld, int col0) {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            double u0, v0, u1, v1;
            uv(4 * j + c, u0, v0);
            uv(4 * j + 2 + c, u1, v1);
            double s = u0 + u1, q = v0 + v1;
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
                s += __shfl_xor_sync(0xffffffffu, s, o);
                q += __shfl_xor_sync(0xffffffffu, q, o);
            }
            if (l < 4) { red[w * 128 + fcol(j, c)] = s; red[512 + w * 128 + fcol(j, c)] = q; }
        }
    __syncthreads();
    const int n = threadIdx.x;
    ps[col0 + n] = ((red[n] + red[128 + n]) + red[256 + n]) + red[384 + n];
    ps[ld + col0 + n] = ((red[512 + n] + red[640 + n]) + red[768 + n]) + red[896 + n];
}

__device__ __forceinline__ void better_max(float& v, int& i, float v2, int i2) { if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; } }
__device__ __forceinline__ void better_min(float& v, int& i, float v2, int i2) { if (v2 < v || (v2 == v && i2 < i)) { v = v2; i = i2; } }

struct FwdArgs {
    const float* x; int R, K;
    const float* tab_in;    // (6, K) table of the input's layer (act applied on load), or null: x as given
    const float* w;         // (N, K)
    int N;
    const float* shift; int gsize;   // (R / gsize, N) added to every row of a group, or null
    float* z;               // (R, N)
    double* ps;             // (R / 64, 2, N)
    float* ev; int* ei;     // (R / 64, 2, N) [max, min] z of the tile and its row within the group, or null
};

template <int MODE>
__global__ void __launch_bounds__(NTH) k_pm_fwd(FwdArgs a) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char* sm = smem_base(smem_raw);
    const int tile = blockIdx.x, n0 = blockIdx.y * TN, tid = threadIdx.x;
    const long long row0 = (long long)tile * TM;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    const int kq = (tid & 7) * 4, rq = tid >> 3;        // vector staging: 4 consecutive k of rows rq + 16 i
    gemm_loop<MODE>(acc, sm, (a.K + KC - 1) / KC, [&](float* As, float* Bs, int c) {
        const int kc = c * KC;
        if (a.K % 4 == 0) {
            const int k = kc + kq;
            const bool ok = k < a.K;
            float4 ta = make_float4(0.f, 0.f, 0.f, 0.f), tb = ta;
            if (ok && a.tab_in) { ta = ld4(a.tab_in + T_A * a.K + k); tb = ld4(a.tab_in + T_B * a.K + k); }
#pragma unroll
            for (int i = 0; i < TM / 16; ++i) {
                const int r = rq + 16 * i;
                float4 v = ok ? ld4(a.x + (row0 + r) * a.K + k) : make_float4(0.f, 0.f, 0.f, 0.f);
                if (ok && a.tab_in) v = act4(v, ta, tb);
                st4(As, r, kq, opnd4<MODE>(v));
            }
#pragma unroll
            for (int i = 0; i < TN / 16; ++i) {
                const int n = rq + 16 * i;
                st4(Bs, n, kq, opnd4<MODE>(ok ? ld4(a.w + (long long)(n0 + n) * a.K + k) : make_float4(0.f, 0.f, 0.f, 0.f)));
            }
            return;
        }
        for (int e = tid; e < TM * KC; e += NTH) {          // a row length that is not a multiple of 4 (the raw points)
            const int r = e >> 5, k = kc + (e & 31);
            float v = 0.f;
            if (k < a.K) {
                v = a.x[(row0 + r) * a.K + k];
                if (a.tab_in) v = fmaxf(fmaf(a.tab_in[T_A * a.K + k], v, a.tab_in[T_B * a.K + k]), 0.f);
            }
            As[swz(r, e & 31)] = opnd<MODE>(v);
        }
        for (int e = tid; e < TN * KC; e += NTH) {
            const int n = e >> 5, k = kc + (e & 31);
            Bs[swz(n, e & 31)] = opnd<MODE>(k < a.K ? a.w[(long long)(n0 + n) * a.K + k] : 0.f);
        }
    });
    if (a.shift) {
        const float* sh = a.shift + (row0 / a.gsize) * a.N + n0;
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) { acc[4 * j + c] += sh[fcol(j, c)]; acc[4 * j + 2 + c] += sh[fcol(j, c)]; }
    }
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int r = 0; r < 2; ++r)
            *reinterpret_cast<float2*>(a.z + (row0 + frow(r)) * a.N + n0 + fcol(j, 0)) = make_float2(acc[4 * j + 2 * r], acc[4 * j + 2 * r + 1]);
    __syncthreads();
    double* red = reinterpret_cast<double*>(sm);
    tile_sums([&](int i, double& u, double& v) { u = acc[i]; v = (double)acc[i] * acc[i]; }, red, a.ps + (size_t)tile * 2 * a.N, a.N, n0);
    if (!a.ev) return;
    __syncthreads();
    float* rv = reinterpret_cast<float*>(sm);
    int* ri = reinterpret_cast<int*>(sm + 4096);
    const int w = tid >> 5, l = tid & 31;
    const int lrow0 = (int)(row0 % a.gsize);
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            // rows ascend with r: the first of equal values keeps the lowest row
            float mx = acc[4 * j + c], mn = mx;
            int ix = frow(0), in = ix;
            better_max(mx, ix, acc[4 * j + 2 + c], frow(1));
            better_min(mn, in, acc[4 * j + 2 + c], frow(1));
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
                better_max(mx, ix, __shfl_xor_sync(0xffffffffu, mx, o), __shfl_xor_sync(0xffffffffu, ix, o));
                better_min(mn, in, __shfl_xor_sync(0xffffffffu, mn, o), __shfl_xor_sync(0xffffffffu, in, o));
            }
            if (l < 4) {
                const int o = w * 128 + fcol(j, c);
                rv[o] = mx; ri[o] = ix; rv[512 + o] = mn; ri[512 + o] = in;
            }
        }
    __syncthreads();
    float mx = rv[tid], mn = rv[512 + tid];
    int ix = ri[tid], in = ri[512 + tid];
    for (int q = 1; q < 4; ++q) { better_max(mx, ix, rv[q * 128 + tid], ri[q * 128 + tid]); better_min(mn, in, rv[512 + q * 128 + tid], ri[512 + q * 128 + tid]); }
    const size_t o = (size_t)tile * 2 * a.N + n0 + tid;
    a.ev[o] = mx; a.ei[o] = lrow0 + ix; a.ev[o + a.N] = mn; a.ei[o + a.N] = lrow0 + in;
}

struct DgradArgs {
    Seg s[2]; int nseg; int R, gsize, Kout;
    const float* zlow; const float* tablow;   // (R, Kout), (6, Kout): the layer below, whose dH this writes
    float* dh;                                // (R, Kout)
    double* ps;                               // (R / 64, 2, Kout): sum dH, sum dH xhat
};

template <int MODE>
__global__ void __launch_bounds__(NTH) k_pm_dgrad(DgradArgs a) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char* sm = smem_base(smem_raw);
    const int tile = blockIdx.x, n0 = blockIdx.y * TN, tid = threadIdx.x;
    const long long row0 = (long long)tile * TM;
    const long long g = row0 / a.gsize;                 // a tile lies inside one group
    const int lrow0 = (int)(row0 - g * a.gsize);
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    const int c0 = a.s[0].N / KC;
    const int kq = (tid & 7) * 4, rq = tid >> 3;
    gemm_loop<MODE>(acc, sm, c0 + (a.nseg > 1 ? a.s[1].N / KC : 0), [&](float* As, float* Bs, int c) {
        const Seg& s = c < c0 ? a.s[0] : a.s[1];
        const int k = (c < c0 ? c : c - c0) * KC + kq;
        const Quad q = quad(s.tab, s.N, k);
#pragma unroll
        for (int i = 0; i < TM / 16; ++i) {
            const int r = rq + 16 * i;
            st4(As, r, kq, opnd4<MODE>(dz4(s, q, row0 + r, k, g, lrow0 + r)));
        }
#pragma unroll
        for (int i = 0; i < TN / 16; ++i) {
            const int n = rq + 16 * i;
            st4(Bs, n, kq, opnd4<MODE>(ld4(s.wt + (long long)(n0 + n) * s.N + k)));
        }
    });
    // dH_low = dY [a z + b > 0]
    const float* t = a.tablow;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const int n = n0 + fcol(j, c);
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const float z = a.zlow[(row0 + frow(r)) * a.Kout + n];
                float& d = acc[4 * j + 2 * r + c];
                d = fmaf(t[T_A * a.Kout + n], z, t[T_B * a.Kout + n]) > 0.f ? d : 0.f;
            }
        }
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int r = 0; r < 2; ++r)
            *reinterpret_cast<float2*>(a.dh + (row0 + frow(r)) * a.Kout + n0 + fcol(j, 0)) = make_float2(acc[4 * j + 2 * r], acc[4 * j + 2 * r + 1]);
    __syncthreads();
    tile_sums([&](int i, double& u, double& v) {      // xhat_low read again rather than kept in registers
        const int n = n0 + fcol(i >> 2, i & 1);
        const float xh = (a.zlow[(row0 + frow((i >> 1) & 1)) * a.Kout + n] - t[T_MU * a.Kout + n]) * t[T_RS * a.Kout + n];
        u = acc[i];
        v = (double)acc[i] * xh;
    }, reinterpret_cast<double*>(sm), a.ps + (size_t)tile * 2 * a.Kout, a.Kout, n0);
}

struct WgradArgs {
    Seg s; int R, gsize;
    const float* x; int K;      // (R, K) the layer's input (pre-activation z of the layer below, or the points)
    const float* tab_in;        // (6, K) or null
    int rows_per_split;
    float* part;                // (splits, N, K)
};

template <int MODE>
__global__ void __launch_bounds__(NTH) k_pm_wgrad(WgradArgs a) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char* sm = smem_base(smem_raw);
    const int split = blockIdx.x, m0 = blockIdx.y * TM, k0 = blockIdx.z * TN, tid = threadIdx.x;
    const long long r_begin = (long long)split * a.rows_per_split;
    const long long r_end = min((long long)a.R, r_begin + a.rows_per_split);
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    // transposed on the way in: a thread reads four consecutive channels (columns) of a row and stores them down the tile's rows
    const int mq = (tid & 15) * 4, ra = tid >> 4;       // A: channels m0 + mq .. + 3 of rows ra + 8 i
    const int nq = (tid & 31) * 4, rb = tid >> 5;       // B: columns k0 + nq .. + 3 of rows rb + 4 i
    const Quad q = quad(a.s.tab, a.s.N, m0 + mq);
    const bool vec_b = a.K % 4 == 0, ok_b = k0 + nq < a.K;
    float4 ta = make_float4(0.f, 0.f, 0.f, 0.f), tb = ta;
    if (vec_b && ok_b && a.tab_in) { ta = ld4(a.tab_in + T_A * a.K + k0 + nq); tb = ld4(a.tab_in + T_B * a.K + k0 + nq); }
    const int chunks = (int)((r_end - r_begin + KC - 1) / KC);
    gemm_loop<MODE>(acc, sm, chunks, [&](float* As, float* Bs, int c) {
        const long long rc = r_begin + (long long)c * KC;
        const long long g = rc / a.gsize;               // a 32-row chunk lies inside one group
        const int lrc = (int)(rc - g * a.gsize);
#pragma unroll
        for (int i = 0; i < KC / 8; ++i) {
            const int rr = ra + 8 * i;
            const float4 v = opnd4<MODE>(dz4(a.s, q, rc + rr, m0 + mq, g, lrc + rr));
            As[swz(mq, rr)] = v.x; As[swz(mq + 1, rr)] = v.y; As[swz(mq + 2, rr)] = v.z; As[swz(mq + 3, rr)] = v.w;
        }
        if (vec_b) {
#pragma unroll
            for (int i = 0; i < KC / 4; ++i) {
                const int rr = rb + 4 * i;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (ok_b) {
                    v = ld4(a.x + (rc + rr) * a.K + k0 + nq);
                    if (a.tab_in) v = act4(v, ta, tb);
                }
                v = opnd4<MODE>(v);
                Bs[swz(nq, rr)] = v.x; Bs[swz(nq + 1, rr)] = v.y; Bs[swz(nq + 2, rr)] = v.z; Bs[swz(nq + 3, rr)] = v.w;
            }
            return;
        }
        for (int e = tid; e < TN * KC; e += NTH) {          // a row length that is not a multiple of 4 (the raw points)
            const int n = e & (TN - 1), rr = e / TN, k = k0 + n;
            float v = 0.f;
            if (k < a.K) {
                v = a.x[(rc + rr) * a.K + k];
                if (a.tab_in) v = fmaxf(fmaf(a.tab_in[T_A * a.K + k], v, a.tab_in[T_B * a.K + k]), 0.f);
            }
            Bs[swz(n, rr)] = opnd<MODE>(v);
        }
    });
    float* out = a.part + (size_t)split * a.s.N * a.K;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const int k = k0 + fcol(j, c);
            if (k >= a.K) continue;
#pragma unroll
            for (int r = 0; r < 2; ++r) out[(size_t)(m0 + frow(r)) * a.K + k] = acc[4 * j + 2 * r + c];
        }
}

// out[j] = sum over i ascending of x[i * n + j] (float64)
template <class T>
__global__ void k_sum_parts(const T* __restrict__ x, int parts, long long n, double* __restrict__ out) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    double s = 0.0;
    for (int i = 0; i < parts; ++i) s += (double)x[(size_t)i * n + j];
    out[j] = s;
}

// per group g of tpg consecutive tiles: out[g, :] = sum over its tiles ascending of ps[tile, :] (width doubles per tile)
__global__ void k_reduce_tiles(const double* __restrict__ ps, int groups, int tpg, int width, double* __restrict__ out) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= (long long)groups * width) return;
    const int g = (int)(j / width), c = (int)(j % width);
    double s = 0.0;
    for (int t = 0; t < tpg; ++t) s += ps[((size_t)g * tpg + t) * width + c];
    out[j] = s;
}

// per group and channel: the max / min z over the group's tiles ascending, lowest row on ties
__global__ void k_group_ext(const float* __restrict__ ev, const int* __restrict__ ei, int groups, int tpg, int N,
                            float* __restrict__ zext, int* __restrict__ iext) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= (long long)groups * N) return;
    const int g = (int)(j / N), n = (int)(j % N);
    float mx = -INFINITY, mn = INFINITY;
    int ix = 0x7fffffff, in = 0x7fffffff;
    for (int t = 0; t < tpg; ++t) {
        const size_t o = ((size_t)g * tpg + t) * 2 * N + n;
        better_max(mx, ix, ev[o], ei[o]);
        better_min(mn, in, ev[o + N], ei[o + N]);
    }
    zext[j] = mx; iext[j] = ix;
    zext[(size_t)groups * N + j] = mn; iext[(size_t)groups * N + j] = in;
}

// dH = dY [a z + b > 0]; per 64-row tile and column: sum dH, sum dH xhat (rows ascending).  One thread per column.
__global__ void k_pm_dh(const float* __restrict__ dy, const float* __restrict__ z, const float* __restrict__ tab, int N,
                        float* __restrict__ dh, double* __restrict__ ps) {
    const int n = blockIdx.y * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const long long row0 = (long long)blockIdx.x * TM;
    const float A = tab[T_A * N + n], B = tab[T_B * N + n], mu = tab[T_MU * N + n], rs = tab[T_RS * N + n];
    double s = 0.0, q = 0.0;
    for (int r = 0; r < TM; ++r) {
        const size_t o = (size_t)(row0 + r) * N + n;
        const float zz = z[o];
        const float d = fmaf(A, zz, B) > 0.f ? dy[o] : 0.f;
        dh[o] = d;
        s += d;
        q += (double)d * ((zz - mu) * rs);
    }
    ps[(size_t)blockIdx.x * 2 * N + n] = s;
    ps[(size_t)blockIdx.x * 2 * N + N + n] = q;
}

__global__ void k_pm_act(const float* __restrict__ z, const float* __restrict__ tab, long long total, int N, float* __restrict__ y) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(i % N);
        y[i] = fmaxf(fmaf(tab[T_A * N + n], z[i], tab[T_B * N + n]), 0.f);
    }
}

template <class K>
int set_smem(K k) {
    DZ_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    return DZ_OK;
}

int check_mode(const char* fn, int mode) {
    if (mode != DZ_F32 && mode != DZ_TF32) { dz_set_error("%s: mode %d (fp32 or tf32 only)", fn, mode); return DZ_ERR_UNSUPPORTED; }
    return DZ_OK;
}

int check_rows(const char* fn, int R, int gsize) {
    if (R <= 0 || R % TM != 0) { dz_set_error("%s: rows %d must be a positive multiple of %d", fn, R, TM); return DZ_ERR_UNSUPPORTED; }
    if (gsize <= 0 || gsize % TM != 0 || R % gsize != 0) {
        dz_set_error("%s: group size %d must be a positive multiple of %d dividing the rows %d", fn, gsize, TM, R);
        return DZ_ERR_UNSUPPORTED;
    }
    return DZ_OK;
}

int wgrad_splits(int R, int N, int K) {
    const int ctas = (N / TM) * dz_cdiv(K, TN);
    int s = dz_cdiv(2 * DZ_NUM_SMS, ctas);
    const int chunks = R / KC;
    return s < 1 ? 1 : (s > chunks ? chunks : s);
}

}  // namespace

extern "C" int dz_pm_fwd(int mode, const float* x, int R, int K, const float* tab_in, const float* w, int N, const float* shift, int gsize,
                         float* z, double* ps, float* ev, int* ei, dz_stream_t stream) {
    DZ_CHECK_ARG(x && w && z && ps && K >= 1 && (!ev || ei));
    int rc = check_mode("dz_pm_fwd", mode);
    if (rc == DZ_OK) rc = check_rows("dz_pm_fwd", R, gsize);
    if (rc != DZ_OK) return rc;
    if (N <= 0 || N % TN != 0) { dz_set_error("dz_pm_fwd: output channels %d must be a multiple of %d", N, TN); return DZ_ERR_UNSUPPORTED; }
    FwdArgs a{x, R, K, tab_in, w, N, shift, gsize, z, ps, ev, ei};
    dim3 grid(R / TM, N / TN);
    cudaStream_t st = (cudaStream_t)stream;
    if (mode == DZ_F32) {
        if ((rc = set_smem(k_pm_fwd<DZ_F32>)) != DZ_OK) return rc;
        k_pm_fwd<DZ_F32><<<grid, NTH, SMEM_BYTES, st>>>(a);
    } else {
        if ((rc = set_smem(k_pm_fwd<DZ_TF32>)) != DZ_OK) return rc;
        k_pm_fwd<DZ_TF32><<<grid, NTH, SMEM_BYTES, st>>>(a);
    }
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

static Seg make_seg(int N, const float* dh, const int* sel, const float* dsel, const float* z, const float* tab, const float* wt) {
    return Seg{N, dh, sel, dsel, z, tab, wt};
}

static int check_seg(const char* fn, const Seg& s, bool need_wt) {
    if (s.N <= 0 || s.N % KC != 0) { dz_set_error("%s: layer channels %d must be a multiple of %d", fn, s.N, KC); return DZ_ERR_UNSUPPORTED; }
    if (!s.z || !s.tab || (!s.dh && !(s.sel && s.dsel)) || (need_wt && !s.wt)) { dz_set_error("%s: missing layer operand", fn); return DZ_ERR_ARG; }
    return DZ_OK;
}

extern "C" int dz_pm_dgrad(int mode, int R, int gsize, int nseg,
                           int N1, const float* dh1, const int* sel1, const float* dsel1, const float* z1, const float* tab1, const float* wt1,
                           int N2, const float* dh2, const int* sel2, const float* dsel2, const float* z2, const float* tab2, const float* wt2,
                           int Kout, const float* zlow, const float* tablow, float* dh, double* ps, dz_stream_t stream) {
    DZ_CHECK_ARG(zlow && tablow && dh && ps && (nseg == 1 || nseg == 2));
    int rc = check_mode("dz_pm_dgrad", mode);
    if (rc == DZ_OK) rc = check_rows("dz_pm_dgrad", R, gsize);
    if (rc != DZ_OK) return rc;
    if (Kout <= 0 || Kout % TN != 0) { dz_set_error("dz_pm_dgrad: input channels %d must be a multiple of %d", Kout, TN); return DZ_ERR_UNSUPPORTED; }
    DgradArgs a{};
    a.s[0] = make_seg(N1, dh1, sel1, dsel1, z1, tab1, wt1);
    a.s[1] = make_seg(N2, dh2, sel2, dsel2, z2, tab2, wt2);
    for (int i = 0; i < nseg; ++i)
        if ((rc = check_seg("dz_pm_dgrad", a.s[i], true)) != DZ_OK) return rc;
    a.nseg = nseg; a.R = R; a.gsize = gsize; a.Kout = Kout; a.zlow = zlow; a.tablow = tablow; a.dh = dh; a.ps = ps;
    dim3 grid(R / TM, Kout / TN);
    cudaStream_t st = (cudaStream_t)stream;
    if (mode == DZ_F32) {
        if ((rc = set_smem(k_pm_dgrad<DZ_F32>)) != DZ_OK) return rc;
        k_pm_dgrad<DZ_F32><<<grid, NTH, SMEM_BYTES, st>>>(a);
    } else {
        if ((rc = set_smem(k_pm_dgrad<DZ_TF32>)) != DZ_OK) return rc;
        k_pm_dgrad<DZ_TF32><<<grid, NTH, SMEM_BYTES, st>>>(a);
    }
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// each row split's partial weight gradient (S, N, K)
static float* carve_wgrad(DzCarve& cv, int R, int N, int K) { return cv.take<float>((size_t)wgrad_splits(R, N, K) * N * K); }

extern "C" size_t dz_pm_wgrad_ws_bytes(int R, int N, int K) { return dz_carve_bytes(carve_wgrad, R, N, K); }

extern "C" int dz_pm_wgrad(int mode, int R, int gsize, int N, const float* dhs, const int* sel, const float* dsel, const float* zs,
                           const float* tab, const float* x, int K, const float* tab_in, double* dw, void* ws, size_t ws_bytes,
                           dz_stream_t stream) {
    DZ_CHECK_ARG(x && dw && ws && K >= 1);
    int rc = check_mode("dz_pm_wgrad", mode);
    if (rc == DZ_OK) rc = check_rows("dz_pm_wgrad", R, gsize);
    if (rc != DZ_OK) return rc;
    if (N <= 0 || N % TM != 0) { dz_set_error("dz_pm_wgrad: output channels %d must be a multiple of %d", N, TM); return DZ_ERR_UNSUPPORTED; }
    WgradArgs a{};
    a.s = make_seg(N, dhs, sel, dsel, zs, tab, nullptr);
    if ((rc = check_seg("dz_pm_wgrad", a.s, false)) != DZ_OK) return rc;
    DZ_CHECK_WS(dz_pm_wgrad_ws_bytes(R, N, K));
    const int S = wgrad_splits(R, N, K);
    DzCarve cv((char*)ws);
    a.part = carve_wgrad(cv, R, N, K);
    a.R = R; a.gsize = gsize; a.x = x; a.K = K; a.tab_in = tab_in;
    a.rows_per_split = dz_cdiv(R / KC, S) * KC;
    dim3 grid(S, N / TM, dz_cdiv(K, TN));
    cudaStream_t st = (cudaStream_t)stream;
    if (mode == DZ_F32) {
        if ((rc = set_smem(k_pm_wgrad<DZ_F32>)) != DZ_OK) return rc;
        k_pm_wgrad<DZ_F32><<<grid, NTH, SMEM_BYTES, st>>>(a);
    } else {
        if ((rc = set_smem(k_pm_wgrad<DZ_TF32>)) != DZ_OK) return rc;
        k_pm_wgrad<DZ_TF32><<<grid, NTH, SMEM_BYTES, st>>>(a);
    }
    DZ_LAUNCH_CHECK();
    const long long n = (long long)N * K;
    k_sum_parts<float><<<dz_cdiv(n, 256), 256, 0, st>>>(a.part, S, n, dw);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" int dz_pm_dh(int R, int N, const float* dy, const float* z, const float* tab, float* dh, double* ps, dz_stream_t stream) {
    DZ_CHECK_ARG(dy && z && tab && dh && ps && N >= 1);
    int rc = check_rows("dz_pm_dh", R, R);
    if (rc != DZ_OK) return rc;
    k_pm_dh<<<dim3(R / TM, dz_cdiv(N, 128)), 128, 0, (cudaStream_t)stream>>>(dy, z, tab, N, dh, ps);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" int dz_pm_act(long long rows, int N, const float* z, const float* tab, float* y, dz_stream_t stream) {
    DZ_CHECK_ARG(z && tab && y && N >= 1 && rows >= 0);
    const long long total = rows * N;
    if (total == 0) return DZ_OK;
    const int blocks = (int)(total / 256 + 1 < 8 * DZ_NUM_SMS ? total / 256 + 1 : 8 * DZ_NUM_SMS);
    k_pm_act<<<blocks, 256, 0, (cudaStream_t)stream>>>(z, tab, total, N, y);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" int dz_pm_reduce_tiles(const double* ps, int groups, int tiles_per_group, int width, double* out, dz_stream_t stream) {
    DZ_CHECK_ARG(ps && out && groups >= 1 && tiles_per_group >= 1 && width >= 1);
    const long long n = (long long)groups * width;
    k_reduce_tiles<<<dz_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(ps, groups, tiles_per_group, width, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" int dz_pm_group_ext(const float* ev, const int* ei, int groups, int tiles_per_group, int N, float* zext, int* iext,
                               dz_stream_t stream) {
    DZ_CHECK_ARG(ev && ei && zext && iext && groups >= 1 && tiles_per_group >= 1 && N >= 1);
    const long long n = (long long)groups * N;
    k_group_ext<<<dz_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(ev, ei, groups, tiles_per_group, N, zext, iext);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// refine_train.cu -- CRM (ConfidencePointnet) point encoders in TRAIN mode, forward and backward, recomputing instead of storing.
//
// Replaces, for refining/detzero_refine/models/modules/confidence_pointnet.py:80-92 in training (pts_encoder_1 -> max over the
// crop's points -> concat -> pts_encoder_2 -> max over points, four 1x1 Conv2d + BatchNorm2d(batch statistics) + ReLU layers) and
// the autograd backward PyTorch runs for it:
//   dz_crm_point_pass      one pass over all B*L*P point rows (see the pass list below), its per-CTA partials reduced in a fixed
//                          order in float64
//
// Layers (C0 -> 128 -> 128 -> 256, then [g | y2] 384 -> 256):  z_l = in_l W_l^T,  y_l = ReLU(a_l z_l + b_l) with a = gamma*rstd,
// b = beta - mean*a from the batch statistics; g = max over the crop of y3; y4 = ReLU(a4 (y2 W4p^T + g W4g^T) + b4), out = max of y4.
// One CTA carries a 64-row tile (inside one crop: P % 64 == 0) through the layers; each layer's output goes through shared memory as
// the next layer's A operand and no (rows, C) activation is ever written to global memory.  Passes:
//   1..4  forward: statistics of z1 / z2 / z3 / z4 (sum and sum of squares, float64); 3 and 4 also keep, per crop and channel, the
//         largest and smallest z and their lowest row (ReLU(a z + b) is monotone in z, so the pooled row is the max row when a >= 0
//         and the min row otherwise); 4 also keeps the per-crop sum of z4 (the crop sums of dz4 follow from it analytically)
//   5     backward: dz4, dz3 (BN backward with the sparse pooled gradient) -> dW4p, dW3 partials, dy2 -> sum dh2, sum dh2*xhat2
//   6     backward: dz2 -> dW2 partials, dy1 -> sum dh1, sum dh1*xhat1
//   7     backward: dz1 -> dW1 partials
// Determinism: every partial is owned by one CTA (grid = min(crops, 132), crops strided over the CTAs), written without atomics,
// and reduced in a fixed order in float64 (k_sum_rows_f64); the same batch gives the same bits.
// Modes: DZ_F32 = exact fp32 FMA; DZ_TF32 = mma.sync m16n8k8 TF32 on the tensor cores (operands rounded to nearest), the arithmetic
// class of the reference's cuDNN 1x1 convs, which run TF32 by default.
#include "common.cuh"

namespace {

constexpr int TM = 64;           // rows per tile
constexpr int NTH = 128;         // threads per CTA
constexpr int C1 = 128, C2 = 128, C3 = 256, C4 = 256, CMAX_IN = 64;
constexpr int LDX = CMAX_IN + 4, LDY = 132, KC = 32, LDW = 136;
constexpr int SMEM_FLOATS = TM * LDX + 3 * TM * LDY + KC * LDW;
constexpr size_t SMEM_BYTES = SMEM_FLOATS * sizeof(float);
// per-layer per-channel table: [a, b, mean, rstd, m1, m2] x 256
enum { T_A = 0, T_B = 1, T_MU = 2, T_RS = 3, T_M1 = 4, T_M2 = 5, T_N = 6 };
constexpr int SLAB = 2 * C4 * C2;  // doubles per CTA: dW4p + dW3 (pass 5) is the largest

struct Args {
    const float* x; int crops, P, c0;
    const float *w1t, *w2t, *w3t, *w4pt;        // K x N (transposed) weights for the forward GEMMs
    const float *w2, *w3, *w4p;                 // N x K (as stored) for the backward dy = dz W
    const float* tab;                           // (4, T_N, 256)
    const float* shift4;                        // (crops, 256) = g W4g^T
    const int* sel;                             // (2, crops, 256) pooled row in the crop, layer 3 then layer 4
    const float* dsel;                          // (2, crops, 256) gradient at the pooled pre-activation (dL/dh), layers 3, 4
    double* stats;                              // (G, 2, 256)
    float* zext; int* iext;                     // (2, crops, 256): [max, min] z and rows (pass 3 / 4)
    double* csum;                               // (crops, 256) per-crop sum of z4 (pass 4)
    double* slab;                               // (G, SLAB)
};

// ---- accumulator layouts: acc[i][j] is output (row(i), col(j)) of a 64 x 128 tile; rows ascend with i --------------------------
template <int MODE> struct Lay;
template <> struct Lay<DZ_F32> {
    static __device__ __forceinline__ int row(int i) { return (threadIdx.x >> 4) + 8 * i; }
    static __device__ __forceinline__ int col(int j) { return (j < 4 ? 0 : 60) + (threadIdx.x & 15) * 4 + j; }
    static __device__ __forceinline__ int rg() { return threadIdx.x >> 4; }
};
template <> struct Lay<DZ_TF32> {
    static __device__ __forceinline__ int row(int i) { return (i >> 1) * 16 + (i & 1) * 8 + ((threadIdx.x & 31) >> 2); }
    static __device__ __forceinline__ int col(int j) { return (threadIdx.x >> 5) * 32 + (j >> 1) * 8 + 2 * (threadIdx.x & 3) + (j & 1); }
    static __device__ __forceinline__ int rg() { return (threadIdx.x & 31) >> 2; }
};

__device__ __forceinline__ uint32_t tf32(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return r;
}

__device__ __forceinline__ void zero(float (&acc)[8][8]) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
}

// acc += A (64 x K) B (K x 128); A(m, k) = AT ? A[k*lda + m] : A[m*lda + k]; B(k, n) = B[k*ldb + n]; all in shared memory, K % 8 == 0
template <int MODE, bool AT>
__device__ __forceinline__ void core(float (&acc)[8][8], const float* A, int lda, const float* B, int ldb, int K) {
    if constexpr (MODE == DZ_F32) {
        const int tr = threadIdx.x >> 4, tc = threadIdx.x & 15;
#pragma unroll 2
        for (int k = 0; k < K; ++k) {
            float a[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) a[i] = AT ? A[k * lda + tr + 8 * i] : A[(tr + 8 * i) * lda + k];
            const float4 b0 = *reinterpret_cast<const float4*>(B + k * ldb + tc * 4);
            const float4 b1 = *reinterpret_cast<const float4*>(B + k * ldb + 64 + tc * 4);
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
    } else {
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
        auto Aat = [&](int m, int k) { return AT ? A[k * lda + m] : A[m * lda + k]; };
        for (int k0 = 0; k0 < K; k0 += 8) {
            uint32_t af[4][4];
#pragma unroll
            for (int mt = 0; mt < 4; ++mt) {
                const int r = mt * 16 + g;
                af[mt][0] = tf32(Aat(r, k0 + t));
                af[mt][1] = tf32(Aat(r + 8, k0 + t));
                af[mt][2] = tf32(Aat(r, k0 + t + 4));
                af[mt][3] = tf32(Aat(r + 8, k0 + t + 4));
            }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int n = w * 32 + nt * 8 + g;
                const uint32_t b0 = tf32(B[(k0 + t) * ldb + n]), b1 = tf32(B[(k0 + t + 4) * ldb + n]);
#pragma unroll
                for (int mt = 0; mt < 4; ++mt) {
                    float* c0 = &acc[mt * 2][nt * 2];
                    float* c1 = &acc[mt * 2 + 1][nt * 2];
                    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                                 : "+f"(c0[0]), "+f"(c0[1]), "+f"(c1[0]), "+f"(c1[1])
                                 : "r"(af[mt][0]), "r"(af[mt][1]), "r"(af[mt][2]), "r"(af[mt][3]), "r"(b0), "r"(b1));
                }
            }
        }
    }
}

// acc += A (64 x K, shared, row-major) W (K x 128 slice of a global K x ldw matrix), W staged through shared memory in KC-row chunks.
// Starts with a barrier, so the caller's last shared-memory writes (A) are visible and earlier readers of Ws are done.
template <int MODE>
__device__ void gemm_w(float (&acc)[8][8], const float* A, int lda, int K, const float* __restrict__ W, int ldw, float* Ws) {
    for (int kc = 0; kc < K; kc += KC) {
        const int kn = min(KC, K - kc);
        __syncthreads();
        for (int e = threadIdx.x; e < kn * 32; e += NTH) {
            const int kk = e >> 5, q = e & 31;
            *reinterpret_cast<float4*>(Ws + kk * LDW + q * 4) = __ldg(reinterpret_cast<const float4*>(W + (size_t)(kc + kk) * ldw + q * 4));
        }
        __syncthreads();
        core<MODE, false>(acc, A + kc, lda, Ws, LDW, kn);
    }
}

// the per-tile column sums of u and v (64 rows; float64), added into the caller's per-thread column accumulators (thread tid owns
// column tid of this 128-column half).  red aliases the D buffer: the caller must be done with it.
template <int MODE, class F>
__device__ __forceinline__ void col_sums(const float (&acc)[8][8], F uv, double* red, double& su, double& sv) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        double s = 0.0, q = 0.0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            double u, v;
            uv(i, j, acc[i][j], u, v);
            s += u;
            q += v;
        }
        red[Lay<MODE>::rg() * 128 + Lay<MODE>::col(j)] = s;
        red[1024 + Lay<MODE>::rg() * 128 + Lay<MODE>::col(j)] = q;
    }
    __syncthreads();
    double s = 0.0, q = 0.0;
    for (int r = 0; r < 8; ++r) { s += red[r * 128 + threadIdx.x]; q += red[1024 + r * 128 + threadIdx.x]; }
    su += s;
    sv += q;
}

__device__ __forceinline__ bool gt(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }
__device__ __forceinline__ bool lt(float v, int i, float bv, int bi) { return v < bv || (v == bv && i < bi); }

// per-tile column max / min of acc with their (lowest) rows, merged into the caller's running extremes of the crop
template <int MODE>
__device__ __forceinline__ void col_ext(const float (&acc)[8][8], int row0, float* red, float& mx, int& ix, float& mn, int& in) {
    __syncthreads();
    int* redi = reinterpret_cast<int*>(red + 2048);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float bx = acc[0][j], bn = acc[0][j];
        int jx = Lay<MODE>::row(0), jn = jx;
#pragma unroll
        for (int i = 1; i < 8; ++i) {        // rows ascend with i: strict comparisons keep the lowest row
            if (acc[i][j] > bx) { bx = acc[i][j]; jx = Lay<MODE>::row(i); }
            if (acc[i][j] < bn) { bn = acc[i][j]; jn = Lay<MODE>::row(i); }
        }
        const int o = Lay<MODE>::rg() * 128 + Lay<MODE>::col(j);
        red[o] = bx; red[1024 + o] = bn; redi[o] = jx; redi[1024 + o] = jn;
    }
    __syncthreads();
    for (int r = 0; r < 8; ++r) {
        const int o = r * 128 + threadIdx.x;
        if (gt(red[o], row0 + redi[o], mx, ix)) { mx = red[o]; ix = row0 + redi[o]; }
        if (lt(red[1024 + o], row0 + redi[1024 + o], mn, in)) { mn = red[1024 + o]; in = row0 + redi[1024 + o]; }
    }
}

// slab[(m0 + row) * ld + col] += acc for col < ncols
template <int MODE>
__device__ __forceinline__ void slab_add(double* slab, int m0, int ld, int ncols, const float (&acc)[8][8]) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = Lay<MODE>::col(j);
            if (n < ncols) slab[(size_t)(m0 + Lay<MODE>::row(i)) * ld + n] += acc[i][j];
        }
}

// store f(acc) (64 x 128) into S (ld LDY); starts with a barrier so earlier readers of S are done
template <int MODE, class F>
__device__ __forceinline__ void store(float* S, const float (&acc)[8][8], F f) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) S[Lay<MODE>::row(i) * LDY + Lay<MODE>::col(j)] = f(i, j, acc[i][j]);
}

// slab[m][n] += sum over the tile's 64 rows of D[row][m] * Bm[row][n], m < 128 (two 64-channel halves), n < ncols
template <int MODE>
__device__ __forceinline__ void wgrad(double* slab, int ld, int ncols, const float* D, const float* Bm, int ldb) {
    __syncthreads();
#pragma unroll 1
    for (int mh = 0; mh < 2; ++mh) {
        float acc[8][8];
        zero(acc);
        core<MODE, true>(acc, D + mh * 64, LDY, Bm, ldb, TM);
        slab_add<MODE>(slab, mh * 64, ld, ncols, acc);
    }
}

template <int MODE, int PASS>
__global__ void __launch_bounds__(NTH, 1) k_crm_point(Args a) {
    extern __shared__ __align__(16) float sm[];
    float* Xs = sm;
    float* Y1 = Xs + TM * LDX;
    float* Y2 = Y1 + TM * LDY;
    float* Ds = Y2 + TM * LDY;
    float* Ws = Ds + TM * LDY;
    double* red = reinterpret_cast<double*>(Ds);          // 2 x 8 x 128 doubles = 16 KB <= the D buffer
    const int tid = threadIdx.x;
    const float* t1 = a.tab;
    const float* t2 = a.tab + 1 * T_N * 256;
    const float* t3 = a.tab + 2 * T_N * 256;
    const float* t4 = a.tab + 3 * T_N * 256;
    double su[2] = {0.0, 0.0}, sv[2] = {0.0, 0.0};
    double* slab = a.slab + (size_t)blockIdx.x * SLAB;
    const int tiles = a.P / TM;

    for (int c = blockIdx.x; c < a.crops; c += gridDim.x) {
        float mx[2], mn[2];
        int ix[2], in[2];
        double cs[2] = {0.0, 0.0};
        for (int h = 0; h < 2; ++h) { mx[h] = -INFINITY; mn[h] = INFINITY; ix[h] = in[h] = 0x7fffffff; }
        for (int tt = 0; tt < tiles; ++tt) {
            const int rloc0 = tt * TM;                            // first row of the tile within the crop
            const float* xg = a.x + ((size_t)c * a.P + rloc0) * a.c0;
            __syncthreads();
            for (int e = tid; e < TM * a.c0 / 4; e += NTH) {
                const int r = e / (a.c0 / 4), q = e % (a.c0 / 4);
                *reinterpret_cast<float4*>(Xs + r * LDX + q * 4) = __ldg(reinterpret_cast<const float4*>(xg + (size_t)r * a.c0 + q * 4));
            }
            float acc[8][8];
            zero(acc);
            gemm_w<MODE>(acc, Xs, LDX, a.c0, a.w1t, C1, Ws);
            if constexpr (PASS == 1) {
                col_sums<MODE>(acc, [](int, int, float z, double& u, double& v) { u = z; v = (double)z * z; }, red, su[0], sv[0]);
                continue;
            }
            store<MODE>(Y1, acc, [&](int, int j, float z) { const int n = Lay<MODE>::col(j); return fmaxf(fmaf(t1[T_A * 256 + n], z, t1[T_B * 256 + n]), 0.f); });
            zero(acc);
            gemm_w<MODE>(acc, Y1, LDY, C1, a.w2t, C2, Ws);
            if constexpr (PASS == 2) {
                col_sums<MODE>(acc, [](int, int, float z, double& u, double& v) { u = z; v = (double)z * z; }, red, su[0], sv[0]);
                continue;
            }
            store<MODE>(Y2, acc, [&](int, int j, float z) { const int n = Lay<MODE>::col(j); return fmaxf(fmaf(t2[T_A * 256 + n], z, t2[T_B * 256 + n]), 0.f); });
            if constexpr (PASS == 3 || PASS == 4) {
#pragma unroll 1
                for (int h = 0; h < 2; ++h) {
                    zero(acc);
                    gemm_w<MODE>(acc, Y2, LDY, C2, (PASS == 3 ? a.w3t : a.w4pt) + h * 128, C3, Ws);
                    if constexpr (PASS == 4) {
                        const float* sh = a.shift4 + (size_t)c * C4 + h * 128;
#pragma unroll
                        for (int i = 0; i < 8; ++i)
#pragma unroll
                            for (int j = 0; j < 8; ++j) acc[i][j] += sh[Lay<MODE>::col(j)];
                    }
                    double ts = 0.0, tq = 0.0;
                    col_sums<MODE>(acc, [](int, int, float z, double& u, double& v) { u = z; v = (double)z * z; }, red, ts, tq);
                    su[h] += ts;
                    sv[h] += tq;
                    cs[h] += ts;
                    col_ext<MODE>(acc, rloc0, reinterpret_cast<float*>(Ds), mx[h], ix[h], mn[h], in[h]);
                }
                continue;
            }
            // ---- backward: dy2 = dz4 W4p + dz3 W3 ----
            float dy[8][8];
            zero(dy);
#pragma unroll 1
            for (int L = 4; L >= 3; --L) {
                const float* tl = L == 4 ? t4 : t3;
                const int* sl = a.sel + (size_t)(L - 3) * a.crops * 256 + (size_t)c * 256;
                const float* dl = a.dsel + (size_t)(L - 3) * a.crops * 256 + (size_t)c * 256;
#pragma unroll 1
                for (int h = 0; h < 2; ++h) {
                    zero(acc);
                    gemm_w<MODE>(acc, Y2, LDY, C2, (L == 4 ? a.w4pt : a.w3t) + h * 128, C3, Ws);
                    const float* sh = a.shift4 + (size_t)c * C4 + h * 128;
                    store<MODE>(Ds, acc, [&](int i, int j, float z) {
                        const int n = h * 128 + Lay<MODE>::col(j);
                        if (L == 4) z += sh[Lay<MODE>::col(j)];
                        const float xh = (z - tl[T_MU * 256 + n]) * tl[T_RS * 256 + n];
                        const float dh = (rloc0 + Lay<MODE>::row(i) == sl[n]) ? dl[n] : 0.f;
                        return tl[T_A * 256 + n] * (dh - tl[T_M1 * 256 + n] - xh * tl[T_M2 * 256 + n]);
                    });
                    if constexpr (PASS == 5) wgrad<MODE>(slab + (L == 4 ? 0 : C4 * C2) + h * 128 * C2, C2, C2, Ds, Y2, LDY);
                    gemm_w<MODE>(dy, Ds, LDY, 128, (L == 4 ? a.w4p : a.w3) + (size_t)h * 128 * C2, C2, Ws);
                }
            }
            zero(acc);
            gemm_w<MODE>(acc, Y1, LDY, C1, a.w2t, C2, Ws);         // z2 again
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int n = Lay<MODE>::col(j);
                    const float z = acc[i][j];
                    dy[i][j] = fmaf(t2[T_A * 256 + n], z, t2[T_B * 256 + n]) > 0.f ? dy[i][j] : 0.f;    // dh2
                    acc[i][j] = (z - t2[T_MU * 256 + n]) * t2[T_RS * 256 + n];                           // xhat2
                }
            if constexpr (PASS == 5) {
                col_sums<MODE>(dy, [&](int i, int j, float d, double& u, double& v) { u = d; v = (double)d * acc[i][j]; }, red, su[0], sv[0]);
                continue;
            }
            store<MODE>(Ds, dy, [&](int i, int j, float d) {
                const int n = Lay<MODE>::col(j);
                return t2[T_A * 256 + n] * (d - t2[T_M1 * 256 + n] - acc[i][j] * t2[T_M2 * 256 + n]);       // dz2
            });
            if constexpr (PASS == 6) wgrad<MODE>(slab, C1, C1, Ds, Y1, LDY);
            zero(dy);
            gemm_w<MODE>(dy, Ds, LDY, C2, a.w2, C1, Ws);           // dy1 = dz2 W2
            zero(acc);
            gemm_w<MODE>(acc, Xs, LDX, a.c0, a.w1t, C1, Ws);       // z1 again
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int n = Lay<MODE>::col(j);
                    const float z = acc[i][j];
                    dy[i][j] = fmaf(t1[T_A * 256 + n], z, t1[T_B * 256 + n]) > 0.f ? dy[i][j] : 0.f;    // dh1
                    acc[i][j] = (z - t1[T_MU * 256 + n]) * t1[T_RS * 256 + n];                           // xhat1
                }
            if constexpr (PASS == 6) {
                col_sums<MODE>(dy, [&](int i, int j, float d, double& u, double& v) { u = d; v = (double)d * acc[i][j]; }, red, su[0], sv[0]);
                continue;
            }
            store<MODE>(Ds, dy, [&](int i, int j, float d) {
                const int n = Lay<MODE>::col(j);
                return t1[T_A * 256 + n] * (d - t1[T_M1 * 256 + n] - acc[i][j] * t1[T_M2 * 256 + n]);       // dz1
            });
            wgrad<MODE>(slab, a.c0, a.c0, Ds, Xs, LDX);           // dW1 (128 x c0)
        }
        if constexpr (PASS == 3 || PASS == 4) {
            const size_t o = (size_t)c * 256;
            for (int h = 0; h < 2; ++h) {
                const int n = h * 128 + tid;
                a.zext[o + n] = mx[h]; a.iext[o + n] = ix[h];
                a.zext[(size_t)a.crops * 256 + o + n] = mn[h]; a.iext[(size_t)a.crops * 256 + o + n] = in[h];
                if (PASS == 4) a.csum[o + n] = cs[h];
            }
        }
    }
    if constexpr (PASS <= 6) {
        for (int h = 0; h < 2; ++h) {
            a.stats[(size_t)blockIdx.x * 512 + h * 128 + tid] = su[h];
            a.stats[(size_t)blockIdx.x * 512 + 256 + h * 128 + tid] = sv[h];
        }
    }
}

template <int MODE>
int launch(int pass, const Args& a, int G, cudaStream_t st) {
    void (*k)(Args) = nullptr;
    switch (pass) {
        case 1: k = k_crm_point<MODE, 1>; break;
        case 2: k = k_crm_point<MODE, 2>; break;
        case 3: k = k_crm_point<MODE, 3>; break;
        case 4: k = k_crm_point<MODE, 4>; break;
        case 5: k = k_crm_point<MODE, 5>; break;
        case 6: k = k_crm_point<MODE, 6>; break;
        case 7: k = k_crm_point<MODE, 7>; break;
        default: dz_set_error("dz_crm_point_pass: pass %d is not 1..7", pass); return DZ_ERR_ARG;
    }
    DZ_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
    k<<<G, NTH, SMEM_BYTES, st>>>(a);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// out[j] = sum over i ascending of x[i * ld + j], j < n
__global__ void k_sum_rows_f64(const double* __restrict__ x, int rows, long long ld, long long n, double* __restrict__ out) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    double s = 0.0;
    for (int i = 0; i < rows; ++i) s += x[(size_t)i * ld + j];
    out[j] = s;
}

}  // namespace

static int crm_point_grid(int crops) { return crops < DZ_NUM_SMS ? crops : DZ_NUM_SMS; }

// each CTA's partials: its 512 BatchNorm sums and its slab
struct CrmWs { double *stats, *slab; };

static CrmWs carve_crm(DzCarve& cv, int crops) {
    const int G = crm_point_grid(crops);
    CrmWs w;
    w.stats = cv.take<double>((size_t)G * 512); w.slab = cv.take<double>((size_t)G * SLAB);
    return w;
}

extern "C" size_t dz_crm_point_ws_bytes(int crops) { return dz_carve_bytes(carve_crm, crops); }

extern "C" int dz_crm_point_pass(int pass, int mode, const float* x, int crops, int P, int c0,
                                 const float* w1t, const float* w2t, const float* w3t, const float* w4pt,
                                 const float* w2, const float* w3, const float* w4p, const float* tab, const float* shift4,
                                 const int* sel, const float* dsel, float* zext, int* iext, double* csum,
                                 double* stats, double* slab, void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(x && crops >= 1 && tab && w1t && ws);
    if (P % TM != 0 || P <= 0) { dz_set_error("dz_crm_point_pass: points per crop P = %d must be a positive multiple of %d", P, TM); return DZ_ERR_UNSUPPORTED; }
    if (c0 % 8 != 0 || c0 < 8 || c0 > CMAX_IN) { dz_set_error("dz_crm_point_pass: point dims %d must be a multiple of 8 in [8, %d]", c0, CMAX_IN); return DZ_ERR_UNSUPPORTED; }
    if (mode != DZ_F32 && mode != DZ_TF32) { dz_set_error("dz_crm_point_pass: mode %d (fp32 or tf32 only)", mode); return DZ_ERR_UNSUPPORTED; }
    DZ_CHECK_ARG(pass < 2 || w2t);
    DZ_CHECK_ARG(pass < 3 || (w3t && w4pt));
    DZ_CHECK_ARG(pass < 4 || shift4);
    DZ_CHECK_ARG((pass != 3 && pass != 4) || (zext && iext));
    DZ_CHECK_ARG(pass != 4 || csum);
    DZ_CHECK_ARG(pass < 5 || (w2 && w3 && w4p && sel && dsel));
    DZ_CHECK_WS(dz_crm_point_ws_bytes(crops));
    const int G = crm_point_grid(crops);
    DzCarve cv((char*)ws);
    const CrmWs w = carve_crm(cv, crops);
    Args a{x, crops, P, c0, w1t, w2t, w3t, w4pt, w2, w3, w4p, tab, shift4, sel, dsel, w.stats, zext, iext, csum, w.slab};
    cudaStream_t st = (cudaStream_t)stream;
    if (pass >= 5) DZ_CUDA(cudaMemsetAsync(a.slab, 0, (size_t)G * SLAB * sizeof(double), st));
    int rc = mode == DZ_F32 ? launch<DZ_F32>(pass, a, G, st) : launch<DZ_TF32>(pass, a, G, st);
    if (rc != DZ_OK) return rc;
    if (pass <= 6 && stats) {
        k_sum_rows_f64<<<dz_cdiv(512, 256), 256, 0, st>>>(a.stats, G, 512, 512, stats);
        DZ_LAUNCH_CHECK();
    }
    if (pass >= 5 && slab) {
        const long long n = pass == 5 ? SLAB : (long long)C1 * (pass == 6 ? C1 : c0);
        k_sum_rows_f64<<<dz_cdiv(n, 256), 256, 0, st>>>(a.slab, G, SLAB, n, slab);
        DZ_LAUNCH_CHECK();
    }
    return DZ_OK;
}

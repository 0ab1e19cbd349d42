// refine.cu -- refiner (GRM / PRM / CRM) building blocks, exact-fp32 SIMT path, sm_90a.
//
// Replaces, for refining/detzero_refine/models/modules/transformer/multi_head_attention.py:90-295
// (multi_head_attention_forward), decoder.py:48-92 (TransformerDecoderLayer.forward), position_encoding.py,
// ffn.py and the 1x1-conv MLP builders utils/detzero_utils/model_utils.py:81-134:
//   dz_linear_fwd          F.linear / Conv1d(k=1) / Conv2d(k=1) (+ folded BatchNorm + ReLU epilogue)
//   dz_group_max           torch.max over the points of a crop (position_transformer.py:109,118)
//   dz_attention_fwd       bmm(q,k^T) + key_padding masked_fill(-inf) + softmax + bmm(.,v), streamed (flash-style
//                          online softmax): the (B*H, Pq, Pk) score tensor (5.9 GB at B=96) is never materialised
//   dz_layernorm_residual  x + dropout(x2) -> LayerNorm (eval: dropout = identity)
// Token-major (B, P, C) activations replace the reference's (B, C, P) <-> (P, B, C) permute copies.
#include "common.cuh"

// ---------------------------------------------------------------------------------------------------------------
// y[m][n] = act((sum_k x[m][k] w[n][k]) * scale[n] + shift[n])
// ---------------------------------------------------------------------------------------------------------------
static constexpr int LN_BM = 128, LN_BN = 64, LN_BK = 8, LN_THREADS = 256;

__global__ void __launch_bounds__(LN_THREADS) k_linear_f32(const float* __restrict__ x, int M, int K, const float* __restrict__ w, int N,
                                                           const float* __restrict__ scale, const float* __restrict__ shift, int relu,
                                                           float* __restrict__ y, int ldy, const float* __restrict__ gshift, int gsize, int grow0) {
    __shared__ __align__(16) float As[LN_BK][LN_BM + 4];
    __shared__ __align__(16) float Bs[LN_BK][LN_BN + 4];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;     // thread tile 8 rows x 4 cols
    const long long m0 = (long long)blockIdx.x * LN_BM;
    const int n0 = blockIdx.y * LN_BN;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const bool vec = (K & 3) == 0;
    for (int k0 = 0; k0 < K; k0 += LN_BK) {
        {   // A tile: 128 rows x 8 k ; thread -> row tid/2, k-half (tid&1)*4
            int r = tid >> 1, kc = (tid & 1) * 4;
            long long m = m0 + r;
            float v[4] = {0.f, 0.f, 0.f, 0.f};
            if (m < M) {
                const float* src = x + (size_t)m * K + k0 + kc;
                if (vec && k0 + kc + 3 < K) { float4 t = __ldg(reinterpret_cast<const float4*>(src)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
                else { for (int i = 0; i < 4; ++i) if (k0 + kc + i < K) v[i] = __ldg(src + i); }
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) As[kc + i][r] = v[i];
        }
        if (tid < 128) {   // B tile: 64 rows(n) x 8 k
            int r = tid >> 1, kc = (tid & 1) * 4;
            int n = n0 + r;
            float v[4] = {0.f, 0.f, 0.f, 0.f};
            if (n < N) {
                const float* src = w + (size_t)n * K + k0 + kc;
                if (vec && k0 + kc + 3 < K) { float4 t = __ldg(reinterpret_cast<const float4*>(src)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
                else { for (int i = 0; i < 4; ++i) if (k0 + kc + i < K) v[i] = __ldg(src + i); }
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) Bs[kc + i][r] = v[i];
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < LN_BK; ++kk) {
            float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * 8]);
            float4 a1 = *reinterpret_cast<const float4*>(&As[kk][ty * 8 + 4]);
            float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        long long m = m0 + ty * 8 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int n = n0 + tx * 4 + j;
            if (n >= N) continue;
            float v = acc[i][j];
            if (scale) v *= __ldg(scale + n);
            if (shift) v += __ldg(shift + n);
            if (gshift) v += __ldg(gshift + (size_t)((grow0 + m) / gsize) * N + n);
            if (relu) v = fmaxf(v, 0.f);
            y[(size_t)m * ldy + n] = v;
        }
    }
}

int dz_linear_fwd_tc(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift, int relu,
                     float* y, int ldy, int mode, const float* gshift, int gsize, cudaStream_t st);

int dz_linear_fwd_f32_rows(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift, int relu,
                           float* y, int ldy, const float* gshift, int gsize, int grow0, cudaStream_t st) {
    if (M <= 0) return DZ_OK;
    dim3 grid(dz_cdiv(M, LN_BM), dz_cdiv(N, LN_BN));
    k_linear_f32<<<grid, LN_THREADS, 0, st>>>(x, M, K, w, N, scale, shift, relu, y, ldy, gshift, gsize > 0 ? gsize : 1, grow0);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// y[m] = act((x[m] W^T) * scale + shift + gshift[m / gsize]): a linear layer whose input is the concatenation [per-group global
// feature | per-row feature] (the PointNet "concat the max-pooled feature back" step, position_transformer.py:118-123,
// geometry_transformer.py:131-136, confidence_pointnet.py:88-100) without materialising the concatenation: the global half of the
// weight is applied once per GROUP (a tiny GEMM the caller runs first -> gshift (M/gsize, N), already scaled), the per-row half here.
extern "C" int dz_linear_fwd_grouped(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift,
                                     const float* gshift, int gsize, int relu, float* y, int ldy, int mode, dz_stream_t stream) {
    DZ_CHECK_ARG(x && w && y && M >= 0 && K >= 1 && N >= 1 && ldy >= N && (!gshift || gsize >= 1));
    if (M == 0) return DZ_OK;
    if (mode != DZ_F32) return dz_linear_fwd_tc(x, M, K, w, N, scale, shift, relu, y, ldy, mode, gshift, gsize, (cudaStream_t)stream);
    return dz_linear_fwd_f32_rows(x, M, K, w, N, scale, shift, relu, y, ldy, gshift, gsize, 0, (cudaStream_t)stream);
}

int dz_linear_max_fwd_tc(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift, int relu, int group,
                         float* gmax, cudaStream_t st);
__global__ void k_fill_f32(float* __restrict__ y, long long n, float v);

// y (M/group, N) = max over each group of `group` consecutive rows of act((x W^T) * scale + shift): the last layer of a PointNet encoder
// fused with torch.max over the points (model_utils.py:81-134 + position_transformer.py:109,118): the (M, N) activation never touches HBM
extern "C" int dz_linear_max_fwd(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift, int relu,
                                 int group, float* y, int mode, dz_stream_t stream) {
    DZ_CHECK_ARG(x && w && y && M >= 1 && K >= 1 && N >= 1 && group >= 1 && M % group == 0);
    if (mode != DZ_TF32) { dz_set_error("dz_linear_max_fwd: tensor-core mode only (the exact-fp32 path runs dz_linear_fwd + dz_group_max)"); return DZ_ERR_UNSUPPORTED; }
    cudaStream_t st = (cudaStream_t)stream;
    const long long n = (long long)(M / group) * N;
    k_fill_f32<<<dz_cdiv(n, 256), 256, 0, st>>>(y, n, -INFINITY);
    return dz_linear_max_fwd_tc(x, M, K, w, N, scale, shift, relu, group, y, st);
}

extern "C" int dz_linear_fwd(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift,
                             int relu, float* y, int ldy, int mode, dz_stream_t stream) {
    return dz_linear_fwd_grouped(x, M, K, w, N, scale, shift, nullptr, 0, relu, y, ldy, mode, stream);
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void k_group_max(const float* __restrict__ x, int G, int group, int C, float* __restrict__ y) {
    long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= (long long)G * C) return;
    int g = (int)(t / C), c = (int)(t % C);
    const float* p = x + (size_t)g * group * C + c;
    float m = -INFINITY;
    for (int r = 0; r < group; ++r) m = fmaxf(m, __ldg(p + (size_t)r * C));
    y[t] = m;
}

// few groups x many rows (PRM memory encoder: 16 tracks x 9600 keys; GRM: 4096 points): the one-thread-per-(group, channel) kernel
// above runs on G*C/256 CTAs (16!) and took 2.1 ms of an 8 ms refiner step.  Split every group's rows over many CTAs; the max is
// order-independent, so an atomic max (sign-aware integer compare of the float bits, y pre-set to -inf) gives the identical result.
// The branch tests the sign BIT: -0.0 >= 0.f holds, but as a signed int -0.0 is INT_MIN, below every negative float, so a float
// compare would send it to atomicMax and a group whose maximum is -0.0 would keep the -inf fill.
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
    if (__float_as_int(v) >= 0) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}
__global__ void k_fill_f32(float* __restrict__ y, long long n, float v) {
    long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t < n) y[t] = v;
}
static constexpr int GM_ROWS = 64;
__global__ void __launch_bounds__(256) k_group_max_split(const float* __restrict__ x, int group, int C, float* __restrict__ y) {
    const int g = blockIdx.y, r0 = blockIdx.x * GM_ROWS, r1 = min(group, r0 + GM_ROWS);
    const float* p = x + ((size_t)g * group + r0) * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float m = -INFINITY;
        for (int r = 0; r < r1 - r0; ++r) m = fmaxf(m, __ldg(p + (size_t)r * C + c));
        atomic_max_float(y + (size_t)g * C + c, m);
    }
}

extern "C" int dz_group_max(const float* x, int G, int group, int C, float* y, dz_stream_t stream) {
    DZ_CHECK_ARG(x && y && G >= 0 && group >= 1 && C >= 1);
    if (G == 0) return DZ_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if ((long long)G * C < 148LL * 256 * 2 && group >= 4 * GM_ROWS) {
        const long long n = (long long)G * C;
        k_fill_f32<<<dz_cdiv(n, 256), 256, 0, st>>>(y, n, -INFINITY);
        dim3 grid(dz_cdiv(group, GM_ROWS), G);
        k_group_max_split<<<grid, C >= 256 ? 256 : 128, 0, st>>>(x, group, C, y);
    } else {
        k_group_max<<<dz_cdiv((long long)G * C, 256), 256, 0, st>>>(x, G, group, C, y);
    }
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// streaming attention, head_dim 32, exact fp32.  Block = 128 threads = 64 query rows x 2 key-halves.
// ---------------------------------------------------------------------------------------------------------------
static constexpr int AT_BQ = 64, AT_BK = 64, AT_DH = 32;

__global__ void __launch_bounds__(128) k_attention_f32(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk,
                                                       const float* __restrict__ v, int ldv, const unsigned char* __restrict__ kpm,
                                                       int Pq, int Pk, int H, float* __restrict__ out, int ldo) {
    __shared__ float Ks[AT_BK][AT_DH + 1];
    __shared__ float Vs[AT_BK][AT_DH + 1];
    __shared__ unsigned char Ms[AT_BK];
    const int bh = blockIdx.y, b = bh / H, h = bh % H;
    const int q0 = blockIdx.x * AT_BQ;
    const int row = threadIdx.x >> 1, half = threadIdx.x & 1;
    const int qi = q0 + row;
    float qr[AT_DH], o[AT_DH];
#pragma unroll
    for (int d = 0; d < AT_DH; ++d) { qr[d] = 0.f; o[d] = 0.f; }
    if (qi < Pq) {
        const float* qp = q + ((size_t)b * Pq + qi) * ldq + h * AT_DH;
#pragma unroll
        for (int d = 0; d < AT_DH; ++d) qr[d] = __ldg(qp + d);
    }
    float mrow = -INFINITY, lrow = 0.f;
    for (int k0 = 0; k0 < Pk; k0 += AT_BK) {
        __syncthreads();
        for (int t = threadIdx.x; t < AT_BK * AT_DH; t += 128) {
            int kk = t / AT_DH, d = t % AT_DH;
            int ki = k0 + kk;
            float kv = 0.f, vv = 0.f;
            if (ki < Pk) {
                kv = __ldg(k + ((size_t)b * Pk + ki) * ldk + h * AT_DH + d);
                vv = __ldg(v + ((size_t)b * Pk + ki) * ldv + h * AT_DH + d);
            }
            Ks[kk][d] = kv; Vs[kk][d] = vv;
        }
        if (threadIdx.x < AT_BK) {
            int ki = k0 + threadIdx.x;
            Ms[threadIdx.x] = (ki >= Pk) ? 1 : (kpm ? kpm[(size_t)b * Pk + ki] : 0);
        }
        __syncthreads();
        float s[AT_BK / 2];
        float tmax = -INFINITY;
#pragma unroll
        for (int j = 0; j < AT_BK / 2; ++j) {
            int kk = 2 * j + half;
            float acc = 0.f;
#pragma unroll
            for (int d = 0; d < AT_DH; ++d) acc = fmaf(qr[d], Ks[kk][d], acc);
            s[j] = Ms[kk] ? -INFINITY : acc;
            tmax = fmaxf(tmax, s[j]);
        }
        tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
        float mnew = fmaxf(mrow, tmax);
        float corr = (mnew == -INFINITY) ? 1.f : expf(mrow - mnew);      // all masked so far: nothing to rescale
        float psum = 0.f;
#pragma unroll
        for (int d = 0; d < AT_DH; ++d) o[d] *= corr;
#pragma unroll
        for (int j = 0; j < AT_BK / 2; ++j) {
            int kk = 2 * j + half;
            float p = (s[j] == -INFINITY) ? 0.f : expf(s[j] - mnew);
            psum += p;
#pragma unroll
            for (int d = 0; d < AT_DH; ++d) o[d] = fmaf(p, Vs[kk][d], o[d]);
        }
        psum += __shfl_xor_sync(0xffffffffu, psum, 1);
        lrow = lrow * corr + psum;
        mrow = mnew;
    }
    // combine the two halves' partial outputs
#pragma unroll
    for (int d = 0; d < AT_DH; ++d) o[d] += __shfl_xor_sync(0xffffffffu, o[d], 1);
    if (qi < Pq) {
        float inv = 1.f / lrow;                                        // lrow == 0 (every key masked) -> NaN like softmax(-inf)
        float* op = out + ((size_t)b * Pq + qi) * ldo + h * AT_DH;
#pragma unroll
        for (int d = half * (AT_DH / 2); d < (half + 1) * (AT_DH / 2); ++d) op[d] = (lrow == 0.f) ? NAN : o[d] * inv;
    }
}

int dz_attention_fwd_tc(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const unsigned char* kpm,
                        int B, int Pq, int Pk, int H, int dh, float* out, int ldo, int mode, cudaStream_t st);

extern "C" int dz_attention_fwd(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                                const unsigned char* key_padding_mask, int B, int Pq, int Pk, int H, int dh, float* out,
                                int ldo, int mode, dz_stream_t stream) {
    DZ_CHECK_ARG(q && k && v && out && B >= 1 && Pq >= 1 && Pk >= 1 && H >= 1);
    if (dh != AT_DH) { dz_set_error("dz_attention_fwd: head_dim %d unsupported (32)", dh); return DZ_ERR_UNSUPPORTED; }
    if (mode != DZ_F32) return dz_attention_fwd_tc(q, ldq, k, ldk, v, ldv, key_padding_mask, B, Pq, Pk, H, dh, out, ldo, mode, (cudaStream_t)stream);
    dim3 grid(dz_cdiv(Pq, AT_BQ), B * H);
    k_attention_f32<<<grid, 128, 0, (cudaStream_t)stream>>>(q, ldq, k, ldk, v, ldv, key_padding_mask, Pq, Pk, H, out, ldo);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// y = LayerNorm(x + r): one warp per row
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_layernorm_residual(const float* __restrict__ x, const float* __restrict__ r,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                            int M, int C, float* __restrict__ y) {
    int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= M) return;
    const float* xp = x + (size_t)warp * C;
    const float* rp = r ? r + (size_t)warp * C : nullptr;
    float vals[16];                                                  // C <= 512
    int cnt = 0;
    float sum = 0.f;
    for (int c = lane; c < C; c += 32, ++cnt) {
        float t = __ldg(xp + c) + (rp ? __ldg(rp + c) : 0.f);
        vals[cnt] = t; sum += t;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    float mean = sum / C;
    float sq = 0.f;
    for (int i = 0; i < cnt; ++i) { float d = vals[i] - mean; sq = fmaf(d, d, sq); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    float rstd = rsqrtf(sq / C + eps);
    float* yp = y + (size_t)warp * C;
    cnt = 0;
    for (int c = lane; c < C; c += 32, ++cnt) yp[c] = (vals[cnt] - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c);
}

extern "C" int dz_layernorm_residual(const float* x, const float* r, const float* gamma, const float* beta, float eps, int M,
                                     int C, float* y, dz_stream_t stream) {
    DZ_CHECK_ARG(x && gamma && beta && y && M >= 0 && C >= 1 && C <= 512);
    if (M == 0) return DZ_OK;
    k_layernorm_residual<<<dz_cdiv((long long)M * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, r, gamma, beta, eps, M, C, y);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// out = a + b (with_pos_embed, decoder.py:45-46)
__global__ void k_add(const float4* __restrict__ a, const float4* __restrict__ b, size_t n4, float4* __restrict__ out) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        float4 x = __ldg(a + i), y = __ldg(b + i);
        out[i] = make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w);
    }
}

extern "C" int dz_add(const float* a, const float* b, size_t n, float* out, dz_stream_t stream) {
    DZ_CHECK_ARG(a && b && out && n % 4 == 0);
    if (n == 0) return DZ_OK;
    int blocks = (int)((n / 4 + 255) / 256);
    if (blocks > DZ_NUM_SMS * 16) blocks = DZ_NUM_SMS * 16;
    k_add<<<blocks, 256, 0, (cudaStream_t)stream>>>((const float4*)a, (const float4*)b, n / 4, (float4*)out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

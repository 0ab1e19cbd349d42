// bev.cu -- sparse->dense BEV scatter and NHWC conv2d / deconv2d (exact-fp32 SIMT path), sm_90a.
//
// Replaces HeightCompression.forward (height_compression.py:20-25: SparseConvTensor.dense() + reshape), the
// ZeroPad2d+Conv2d+BatchNorm2d+ReLU stacks and ConvTranspose2d deblocks of BaseBEVBackbone
// (backbone2d.py:34-81,89-120) and the conv stacks of CenterHead/SeparateHead (center_head.py:14-48,81-88).
//
// Layout: dense maps are NHWC so that a pixel's channel vector is one contiguous 128-bit-loadable run and the
// implicit-GEMM K dimension (tap, cin) is contiguous; BatchNorm (eval) + bias + ReLU are folded into the epilogue
// and torch.cat of the deblock outputs (backbone2d.py:107-108) is fused as a channel-offset write.
// DZ_F32 here is the exact-fp32 path; the wgmma tensor-core path lives in conv2d_tc.cu.
#include <stdlib.h>
#include "common.cuh"
#include "conv2d.cuh"

// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_sparse_to_bev(const float* __restrict__ feats, const int32_t* __restrict__ coords,
                                                       const int* __restrict__ d_n, int cap, int c, int D, int H, int W,
                                                       float* __restrict__ out) {
    int n = min(*d_n, cap);
    // one warp per site: lanes stride over channels
    int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int i = warp; i < n; i += nwarps) {
        int4 cd = __ldg(reinterpret_cast<const int4*>(coords) + i);            // b,z,y,x
        float* dst = out + (((size_t)cd.x * H + cd.z) * W + cd.w) * ((size_t)c * D) + cd.y;
        for (int ch = lane; ch < c; ch += 32) dst[(size_t)ch * D] = __ldg(feats + (size_t)i * c + ch);   // channel = c*D + z
    }
}

extern "C" int dz_sparse_to_bev(const float* feats, const int32_t* coords, const int* d_n, int cap, int c, int B, int D,
                                int H, int W, float* out, dz_stream_t stream) {
    DZ_CHECK_ARG(feats && coords && d_n && out && cap >= 1 && c >= 1);
    int blocks = max(1, min(dz_cdiv((long long)cap * 32, 256), DZ_NUM_SMS * 8));
    k_sparse_to_bev<<<blocks, 256, 0, (cudaStream_t)stream>>>(feats, coords, d_n, cap, c, D, H, W, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// SIMT implicit-GEMM conv2d: M = B*Ho*Wo output pixels, N = cout, K = KH*KW*cin
// ---------------------------------------------------------------------------------------------------------------

static constexpr int C2_BM = 128, C2_BK = 8, C2_THREADS = 256;

template <int BN, int TN>
__global__ void __launch_bounds__(C2_THREADS) k_conv2d_f32(Conv2dParams p) {
    __shared__ __align__(16) float As[C2_BK][C2_BM + 4];
    __shared__ __align__(16) float Bs[C2_BK][BN];
    const int tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;                  // 16 x 16 threads; thread tile 8 x TN
    const long long M = (long long)p.B * p.Ho * p.Wo;
    const long long m0 = (long long)blockIdx.x * C2_BM;
    const int n0 = blockIdx.y * BN;

    // the pixel this thread loads for the A tile
    const int lp = tid >> 1, lc = (tid & 1) * 4;
    long long lm = m0 + lp;
    bool lvalid = lm < M;
    int lb = 0, ly = 0, lx = 0;
    if (lvalid) { lx = (int)(lm % p.Wo); long long t = lm / p.Wo; ly = (int)(t % p.Ho); lb = (int)(t / p.Ho); }

    float acc[8][TN];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    for (int r = 0; r < p.KH; ++r) {
        for (int s = 0; s < p.KW; ++s) {
            int yi = ly * p.stride - p.pad + r, xi = lx * p.stride - p.pad + s;
            bool inb = lvalid && (unsigned)yi < (unsigned)p.H && (unsigned)xi < (unsigned)p.W;
            const float* arow = p.in + (((size_t)lb * p.H + yi) * p.W + xi) * p.in_cstride;
            const float* wtap = p.w + (size_t)(r * p.KW + s) * p.cin * p.cout;
            for (int c0 = 0; c0 < p.cin; c0 += C2_BK) {
                float4 av = make_float4(0.f, 0.f, 0.f, 0.f);
                if (inb) av = __ldg(reinterpret_cast<const float4*>(arow + c0 + lc));
                As[lc + 0][lp] = av.x; As[lc + 1][lp] = av.y; As[lc + 2][lp] = av.z; As[lc + 3][lp] = av.w;
                for (int t = tid; t < C2_BK * (BN / 4); t += C2_THREADS) {
                    int kk = t / (BN / 4), n4 = (t % (BN / 4)) * 4;
                    float4 wv = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (n0 + n4 < p.cout) wv = __ldg(reinterpret_cast<const float4*>(wtap + (size_t)(c0 + kk) * p.cout + n0 + n4));
                    *reinterpret_cast<float4*>(&Bs[kk][n4]) = wv;
                }
                __syncthreads();
#pragma unroll
                for (int kk = 0; kk < C2_BK; ++kk) {
                    float a[8], b[TN];
                    float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * 8]);
                    float4 a1 = *reinterpret_cast<const float4*>(&As[kk][ty * 8 + 4]);
                    a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
#pragma unroll
                    for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
                    for (int i = 0; i < 8; ++i)
#pragma unroll
                        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
                }
                __syncthreads();
            }
        }
    }
    // epilogue
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        long long m = m0 + ty * 8 + i;
        if (m >= M) continue;
        int x = (int)(m % p.Wo); long long t = m / p.Wo; int y = (int)(t % p.Ho); int b = (int)(t / p.Ho);
        float* orow = p.out + (((size_t)b * p.OH + (y * p.os + p.oy0)) * p.OW + (x * p.os + p.ox0)) * p.out_cstride + p.out_coff;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            int n = n0 + tx * TN + j;
            if (n >= p.cout) continue;
            float v = acc[i][j];
            if (p.scale) v *= __ldg(p.scale + n);
            if (p.shift) v += __ldg(p.shift + n);
            if (p.relu) v = fmaxf(v, 0.f);
            orow[n] = v;
        }
    }
}

static int conv2d_f32_launch(const Conv2dParams& p, cudaStream_t st) {
    long long M = (long long)p.B * p.Ho * p.Wo;
    int gm = dz_cdiv(M, C2_BM);
    if (p.cout >= 128 || p.cout > 64) {
        dim3 grid(gm, dz_cdiv(p.cout, 128));
        k_conv2d_f32<128, 8><<<grid, C2_THREADS, 0, st>>>(p);
    } else if (p.cout > 16) {
        dim3 grid(gm, dz_cdiv(p.cout, 64));
        k_conv2d_f32<64, 4><<<grid, C2_THREADS, 0, st>>>(p);
    } else {
        dim3 grid(gm, 1);
        k_conv2d_f32<16, 1><<<grid, C2_THREADS, 0, st>>>(p);
    }
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

int dz_conv2d_fwd_tc(const Conv2dParams& p, int mode, cudaStream_t st);

// the fp32 kernel reads the input as float4 (and the TMA unit needs a 16-byte aligned base), the tensor-core per-thread epilogue
// writes float2: a view at an odd storage offset is refused rather than faulting on a misaligned vector access
static bool vector_aligned(const float* in, const float* out) {
    return (reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0;
}

extern "C" int dz_conv2d_fwd(const float* in, int B, int H, int W, int cin, int in_cstride, const float* weight, int KH,
                             int KW, int stride, int pad, const float* scale, const float* shift, int relu, float* out,
                             int Ho, int Wo, int cout, int out_coff, int out_cstride, int mode, dz_stream_t stream) {
    DZ_CHECK_ARG(in && weight && out && B >= 1 && cin % C2_BK == 0 && in_cstride % 4 == 0 && cout % 4 == 0);
    DZ_CHECK_ARG(Ho == (H + 2 * pad - KH) / stride + 1 && Wo == (W + 2 * pad - KW) / stride + 1);
    DZ_CHECK_ARG(vector_aligned(in, out));
    Conv2dParams p{in, weight, scale, shift, out, B, H, W, cin, in_cstride, KH, KW, stride, pad, Ho, Wo, cout,
                   Ho, Wo, 1, 0, 0, out_coff, out_cstride, relu};
    if (mode == DZ_F32) return conv2d_f32_launch(p, (cudaStream_t)stream);
    return dz_conv2d_fwd_tc(p, mode, (cudaStream_t)stream);
}

extern "C" int dz_deconv2d_fwd(const float* in, int B, int H, int W, int cin, const float* weight, int s,
                               const float* scale, const float* shift, int relu, float* out, int cout, int out_coff,
                               int out_cstride, int mode, dz_stream_t stream) {
    DZ_CHECK_ARG(in && weight && out && s >= 1 && cin % C2_BK == 0 && cout % 4 == 0);
    DZ_CHECK_ARG(vector_aligned(in, out));
    if (mode != DZ_F32) {
        // tensor cores: one GEMM with N = s * s * cout over the input pixels (weights (dy, dx, cout, cin))
        Conv2dParams p{in, weight, scale, shift, out, B, H, W, cin, cin, 1, 1, 1, 0, H, W, cout, H * s, W * s, s, 0, 0,
                       out_coff, out_cstride, relu};
        return dz_conv2d_fwd_tc(p, mode, (cudaStream_t)stream);
    }
    for (int dy = 0; dy < s; ++dy)
        for (int dx = 0; dx < s; ++dx) {
            Conv2dParams p{in, weight + (size_t)(dy * s + dx) * cin * cout, scale, shift, out, B, H, W, cin, cin,
                           1, 1, 1, 0, H, W, cout, H * s, W * s, s, dy, dx, out_coff, out_cstride, relu};
            int rc = conv2d_f32_launch(p, (cudaStream_t)stream);
            if (rc) return rc;
        }
    return DZ_OK;
}

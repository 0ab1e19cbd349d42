// spconv.cu -- sparse convolution forward (output-stationary implicit GEMM over the neighbour table), sm_90a.
//
// Replaces spconv SubMConv3d / SparseConv3d forward + BatchNorm1d(eval) + bias + residual + ReLU as composed at
// detection/detzero_det/models/centerpoint_modules/backbone3d.py:64-83 (post_act_block) and :105-121
// (SparseBasicBlock.forward).  One launch per layer; features make exactly one HBM round trip per layer
// (the reference makes three: conv, BN, ReLU).
//
// DZ_F32 path (this file): exact-fp32 FMA.  A CTA owns 64 consecutive output rows and keeps their accumulators in
// shared memory; for every kernel offset k the rows that actually have a neighbour are COMPACTED (ballot prefix)
// so FMA work is proportional to the number of rulebook pairs, not to 27 x rows.  Gathered input rows and the
// W[k] slice are staged in shared memory with 128-bit loads.  No atomics: every output row is owned by one CTA
// => deterministic, unlike gather-GEMM-scatter.
#include "common.cuh"

static constexpr int SP_TM = 64;        // output rows per CTA tile
static constexpr int SP_CK = 32;        // input-channel chunk
static constexpr int SP_THREADS = 256;
static constexpr int SP_AS = SP_CK + 4; // padded A row stride (floats) -> conflict-free float4 reads

template <int COUT>
struct SpSmem {
    float acc[(SP_TM + 1) * COUT];      // +1 trash row for list padding
    float a[(SP_TM + 4) * SP_AS];
    float w[SP_CK * COUT];
    int list[SP_TM + 4];
    int idx[SP_TM + 4];
    int m;
};

template <int COUT>
__global__ void __launch_bounds__(SP_THREADS) k_spconv_f32(const float* __restrict__ in, int cin, const int32_t* __restrict__ nbr,
                                                           int K, int nbr_cap, const int* __restrict__ d_n_out, int out_cap,
                                                           const float* __restrict__ weight, const float* __restrict__ scale,
                                                           const float* __restrict__ shift, const float* __restrict__ residual,
                                                           int relu, float* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SpSmem<COUT>& s = *reinterpret_cast<SpSmem<COUT>*>(smem_raw);
    constexpr int CG = COUT / 4;                 // column groups of 4
    constexpr int RL = SP_THREADS / CG;          // row lanes
    const int tid = threadIdx.x;
    const int cg = tid % CG, rl = tid / CG;
    const int n = min(*d_n_out, out_cap);
    const int n_tiles = (n + SP_TM - 1) / SP_TM;
    const bool vec_in = (cin & 3) == 0;

    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int row0 = tile * SP_TM;
        for (int t = tid; t < (SP_TM + 1) * COUT; t += SP_THREADS) s.acc[t] = 0.f;
        __syncthreads();

        for (int k = 0; k < K; ++k) {
            // ---- compact the rows of this tile that have a neighbour through offset k
            if (tid < SP_TM) {
                int r = row0 + tid;
                int j = r < n ? __ldg(nbr + (size_t)k * nbr_cap + r) : -1;
                unsigned bal = __ballot_sync(0xffffffffu, j >= 0);
                int pos = __popc(bal & ((1u << (tid & 31)) - 1u));
                int cnt = __popc(bal);
                if ((tid & 31) == 0) s.idx[SP_TM + (tid >> 5)] = cnt;      // scratch: warp counts
                __syncwarp();
                // both warps need the first warp's count
                asm volatile("bar.sync 1, 64;");
                int base = (tid >> 5) ? s.idx[SP_TM] : 0;
                int m = s.idx[SP_TM] + s.idx[SP_TM + 1];
                asm volatile("bar.sync 1, 64;");
                if (j >= 0) { s.list[base + pos] = tid; s.idx[base + pos] = j; }
                if (tid == 0) s.m = m;
                asm volatile("bar.sync 1, 64;");
                int m4 = (m + 3) & ~3;
                if (tid >= m && tid < m4) { s.list[tid] = SP_TM; s.idx[tid] = -1; }
            }
            __syncthreads();
            const int m = s.m;
            if (m == 0) { __syncthreads(); continue; }
            const int m4 = (m + 3) & ~3;

            for (int c0 = 0; c0 < cin; c0 += SP_CK) {
                const int ck = min(SP_CK, cin - c0);
                // ---- stage gathered A rows (m4 x SP_CK) and W[k][c0:c0+CK][:] in smem
                if (vec_in) {
                    for (int t = tid; t < m4 * (SP_CK / 4); t += SP_THREADS) {
                        int rs = t / (SP_CK / 4), c4 = (t % (SP_CK / 4)) * 4;
                        int j = s.idx[rs];
                        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (j >= 0 && c4 < ck) v = __ldg(reinterpret_cast<const float4*>(in + (size_t)j * cin + c0 + c4));
                        *reinterpret_cast<float4*>(&s.a[rs * SP_AS + c4]) = v;
                    }
                } else {
                    for (int t = tid; t < m4 * SP_CK; t += SP_THREADS) {
                        int rs = t / SP_CK, c = t % SP_CK;
                        int j = s.idx[rs];
                        s.a[rs * SP_AS + c] = (j >= 0 && c < ck) ? __ldg(in + (size_t)j * cin + c0 + c) : 0.f;
                    }
                }
                const float* wk = weight + ((size_t)k * cin + c0) * COUT;
                for (int t = tid; t < SP_CK * CG; t += SP_THREADS) {
                    int c = t / CG, g4 = (t % CG) * 4;
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (c < ck) v = __ldg(reinterpret_cast<const float4*>(wk + (size_t)c * COUT + g4));
                    *reinterpret_cast<float4*>(&s.w[c * COUT + g4]) = v;
                }
                __syncthreads();
                // ---- FMA: thread owns 4 row-slots x 4 columns
                for (int rs4 = rl * 4; rs4 < m4; rs4 += RL * 4) {
                    float4 acc4[4];
#pragma unroll
                    for (int r = 0; r < 4; ++r) acc4[r] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int c = 0; c < SP_CK; c += 4) {
                        float4 w0 = *reinterpret_cast<const float4*>(&s.w[(c + 0) * COUT + cg * 4]);
                        float4 w1 = *reinterpret_cast<const float4*>(&s.w[(c + 1) * COUT + cg * 4]);
                        float4 w2 = *reinterpret_cast<const float4*>(&s.w[(c + 2) * COUT + cg * 4]);
                        float4 w3 = *reinterpret_cast<const float4*>(&s.w[(c + 3) * COUT + cg * 4]);
#pragma unroll
                        for (int r = 0; r < 4; ++r) {
                            float4 a = *reinterpret_cast<const float4*>(&s.a[(rs4 + r) * SP_AS + c]);
                            acc4[r].x = fmaf(a.x, w0.x, acc4[r].x); acc4[r].y = fmaf(a.x, w0.y, acc4[r].y);
                            acc4[r].z = fmaf(a.x, w0.z, acc4[r].z); acc4[r].w = fmaf(a.x, w0.w, acc4[r].w);
                            acc4[r].x = fmaf(a.y, w1.x, acc4[r].x); acc4[r].y = fmaf(a.y, w1.y, acc4[r].y);
                            acc4[r].z = fmaf(a.y, w1.z, acc4[r].z); acc4[r].w = fmaf(a.y, w1.w, acc4[r].w);
                            acc4[r].x = fmaf(a.z, w2.x, acc4[r].x); acc4[r].y = fmaf(a.z, w2.y, acc4[r].y);
                            acc4[r].z = fmaf(a.z, w2.z, acc4[r].z); acc4[r].w = fmaf(a.z, w2.w, acc4[r].w);
                            acc4[r].x = fmaf(a.w, w3.x, acc4[r].x); acc4[r].y = fmaf(a.w, w3.y, acc4[r].y);
                            acc4[r].z = fmaf(a.w, w3.z, acc4[r].z); acc4[r].w = fmaf(a.w, w3.w, acc4[r].w);
                        }
                    }
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        int row = s.list[rs4 + r];
                        float4* p = reinterpret_cast<float4*>(&s.acc[row * COUT + cg * 4]);
                        float4 o = *p;
                        o.x += acc4[r].x; o.y += acc4[r].y; o.z += acc4[r].z; o.w += acc4[r].w;
                        *p = o;
                    }
                }
                __syncthreads();
            }
        }
        // ---- epilogue: folded BN / bias, residual, ReLU
        for (int t = tid; t < SP_TM * CG; t += SP_THREADS) {
            int row = t / CG, g4 = (t % CG) * 4;
            int r = row0 + row;
            if (r >= n) continue;
            float4 v = *reinterpret_cast<const float4*>(&s.acc[row * COUT + g4]);
            if (scale) {
                float4 sc = __ldg(reinterpret_cast<const float4*>(scale + g4));
                v.x *= sc.x; v.y *= sc.y; v.z *= sc.z; v.w *= sc.w;
            }
            if (shift) {
                float4 sh = __ldg(reinterpret_cast<const float4*>(shift + g4));
                v.x += sh.x; v.y += sh.y; v.z += sh.z; v.w += sh.w;
            }
            if (residual) {
                float4 rr = __ldg(reinterpret_cast<const float4*>(residual + (size_t)r * COUT + g4));
                v.x += rr.x; v.y += rr.y; v.z += rr.z; v.w += rr.w;
            }
            if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
            *reinterpret_cast<float4*>(out + (size_t)r * COUT + g4) = v;
        }
        __syncthreads();
    }
}

template <int COUT>
static int launch_f32(const float* in, int cin, const int32_t* nbr, int K, int nbr_cap, const int* d_n_out, int out_cap,
                      const float* weight, const float* scale, const float* shift, const float* residual, int relu,
                      float* out, cudaStream_t st) {
    size_t smem = sizeof(SpSmem<COUT>);
    static bool configured = false;
    if (!configured) {
        DZ_CUDA(cudaFuncSetAttribute(k_spconv_f32<COUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = true;
    }
    int tiles = dz_cdiv(out_cap, SP_TM);
    int occ = (int)(200 * 1024 / smem); if (occ < 1) occ = 1; if (occ > 6) occ = 6;
    int blocks = max(1, min(tiles, DZ_NUM_SMS * occ));
    k_spconv_f32<COUT><<<blocks, SP_THREADS, smem, st>>>(in, cin, nbr, K, nbr_cap, d_n_out, out_cap, weight, scale, shift,
                                                         residual, relu, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// DZ_TF32 / DZ_TF32X3: csrc/spconv_tc.cu
int dz_spconv_fwd_tc(const float* in, int cin, int in_rows, const int32_t* nbr, int K, int nbr_cap, const int32_t* order, const int* d_n_out, int out_cap,
                     const float* weight, const float* scale, const float* shift, const float* residual, int relu,
                     float* out, int cout, int mode, cudaStream_t st);

extern "C" int dz_spconv_fwd(const float* in, int cin, int in_rows, const int32_t* nbr, int K, int nbr_cap, const int32_t* row_order, const int* d_n_out,
                             int out_cap, const float* weight, const float* scale, const float* shift,
                             const float* residual, int relu, float* out, int cout, int mode, dz_stream_t stream) {
    DZ_CHECK_ARG(in && nbr && d_n_out && weight && out && cin >= 1 && K >= 1 && out_cap >= 1 && nbr_cap >= out_cap);
    cudaStream_t st = (cudaStream_t)stream;
    if (mode == DZ_F32) {
        if (row_order) { dz_set_error("dz_spconv_fwd: row_order is for the tensor-core modes (the fp32 kernel compacts per offset itself)"); return DZ_ERR_UNSUPPORTED; }
        switch (cout) {
            case 16: return launch_f32<16>(in, cin, nbr, K, nbr_cap, d_n_out, out_cap, weight, scale, shift, residual, relu, out, st);
            case 32: return launch_f32<32>(in, cin, nbr, K, nbr_cap, d_n_out, out_cap, weight, scale, shift, residual, relu, out, st);
            case 64: return launch_f32<64>(in, cin, nbr, K, nbr_cap, d_n_out, out_cap, weight, scale, shift, residual, relu, out, st);
            case 128: return launch_f32<128>(in, cin, nbr, K, nbr_cap, d_n_out, out_cap, weight, scale, shift, residual, relu, out, st);
            default: dz_set_error("dz_spconv_fwd: cout=%d unsupported (16/32/64/128)", cout); return DZ_ERR_UNSUPPORTED;
        }
    }
    return dz_spconv_fwd_tc(in, cin, in_rows, nbr, K, nbr_cap, row_order, d_n_out, out_cap, weight, scale, shift, residual, relu, out, cout, mode, st);
}

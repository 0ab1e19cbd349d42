// conv2d_tc.cu -- NHWC conv2d as a wgmma implicit GEMM (TF32 inputs, fp32 register accumulation), sm_90a.
//
// Replaces the cuDNN convolutions of BaseBEVBackbone / CenterHead (backbone2d.py:34-81, center_head.py:25-31,81-88);
// the reference runs them with TF32 tensor cores too (torch.backends.cudnn.allow_tf32 defaults to True, SURVEY A.6).
//
// Design: output tile = 8 x 16 pixel patch (M = 128) x BN output channels.  For every filter tap (r,s) and every
// 32-channel slice of Cin, ONE 4-D TMA box load of the shifted input patch lands in shared memory already in the
// canonical K-major 128B-swizzled layout (row = pixel, 128 B = 32 fp32 channels); out-of-image pixels are
// zero-filled by the TMA unit, which implements the conv padding (and ZeroPad2d) for free.  Weights are a 2-D TMA
// load of W[cout][(r,s,cin)].  Two consumer warpgroups (64 pixels each) issue wgmma (M=64, N=BN, K=8) into register
// accumulators; a ring of mbarrier-guarded stages overlaps TMA with MMA.  After the main loop the accumulators go to a
// shared-memory tile and the same 8 warps run the epilogue (each one quarter of the pixels and half of the channels):
// folded BatchNorm / bias / ReLU, NHWC rows written through TMA stores (optionally into a channel slice / strided pixels:
// fused torch.cat and ConvTranspose2d with kernel == stride), or a fused max over row groups.
#include <stdlib.h>
#include "common.cuh"
#include "conv2d.cuh"
#include "tc.cuh"

namespace tc {
EncodeTiledFn get_encode_tiled() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}
}  // namespace tc

static constexpr int CT_TH = 8, CT_TW = 16, CT_BK = 32;       // pixel patch, channels per k-step group (128 B)
static constexpr int CT_A_BYTES = CT_TH * CT_TW * CT_BK * 4;  // 16 KB
static constexpr int CT_CONSUMERS = 8;                        // warps 0-7: two wgmma warpgroups, then the epilogue
static constexpr int CT_THREADS = 32 * (CT_CONSUMERS + 1);    // warp 8: TMA producer

// HALO variant (3x3 stride-1 convolutions, 16 of the 22 dense convs of the BEV backbone + head).  The generic kernel re-reads its
// 128-pixel activation patch from L2 once per filter tap: 9 x 16 KB per 32-channel slice.  The halo kernel loads the (16+2) x (8+2)
// pixel HALO of a 16 x 8 output patch ONCE per 32-channel slice (23 KB) and the nine taps are nine A descriptors into that one tile:
// a K-major SW128 descriptor may start at any 128-byte pixel row, its 8-row core groups are the 8-pixel rows of the patch, and the
// stride between groups (SBO) is the halo's row pitch, 10 pixels = 1280 B.  The 128-byte swizzle is a function of the absolute
// shared-memory address for the TMA unit and for wgmma alike, so a window shifted by (r, s) reads exactly the bytes the TMA unit wrote
// for pixel (y + r, x + s) with the descriptor's base-offset field left at 0 (measured: the field set to (start >> 7) & 7 gives
// wrong results; the conv2d tests cover every tile width).
static constexpr int HL_TH = 16, HL_TW = 8, HL_PITCH = HL_TW + 2, HL_ROWS = HL_TH + 2;
static constexpr int HL_A_BYTES = HL_ROWS * HL_PITCH * 128;          // 23040 B delivered by the TMA unit
static constexpr int HL_A_SLOT = (HL_A_BYTES + 1023) / 1024 * 1024;  // 23552: slots stay 1024-byte aligned (swizzle phase)
static constexpr int HL_A_STAGES = 2;

template <int BN, bool HALO>
struct CtCfg {
    static constexpr int TH = HALO ? HL_TH : CT_TH, TW = HALO ? HL_TW : CT_TW;        // output patch (TH x TW = 128 pixels)
    static constexpr int B_BYTES = BN * CT_BK * 4;
    static constexpr int ACC_LD = BN + 4;                               // row pitch of the staged accumulator tile
    static constexpr int ACC_BYTES = CT_TH * CT_TW * ACC_LD * 4;
    static constexpr int BUDGET = 227 * 1024 - 1024 - 256 - ACC_BYTES;  // H100: 227 KB of shared memory per block
    // generic: STAGES x (A patch + B tile); halo: HL_A_STAGES halo slots + STAGES B tiles
    static constexpr int STAGE_BYTES = HALO ? B_BYTES : CT_A_BYTES + B_BYTES;
    static constexpr int A_REGION = HALO ? HL_A_STAGES * HL_A_SLOT : 0;
    static constexpr int FIT = (BUDGET - A_REGION) / STAGE_BYTES;
    static constexpr int STAGES = FIT > (HALO ? 9 : 8) ? (HALO ? 9 : 8) : FIT;
    static constexpr int BUF = A_REGION + STAGES * STAGE_BYTES;         // pipeline buffers (epilogue staging slots afterwards)
    static constexpr int SMEM = BUF + ACC_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

__device__ long long g_ct_trace[64];          // DZ_CONV2D_DBG & 4: clock stamps of CTA 0 (dz_debug_conv2d_trace)
extern "C" int dz_debug_conv2d_trace(long long* host) {
    cudaDeviceSynchronize();
    return cudaMemcpyFromSymbol(host, g_ct_trace, sizeof(long long) * 64) == cudaSuccess ? 0 : -1;
}

template <int BN, bool HALO>
__global__ void __launch_bounds__(CT_THREADS, 1)
k_conv2d_tf32(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
              Conv2dParams p, int tiles_x, int tiles_y) {
    using Cfg = CtCfg<BN, HALO>;
    constexpr int TH = Cfg::TH, TW = Cfg::TW;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* smB = smem + Cfg::A_REGION;                              // halo: the B ring follows the halo slots
    float* acc_stg = reinterpret_cast<float*>(smem + Cfg::BUF);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::BUF + Cfg::ACC_BYTES);
    uint64_t* empty = full + Cfg::STAGES;
    uint64_t* a_full = empty + Cfg::STAGES;                                 // halo slots
    uint64_t* a_empty = a_full + HL_A_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool tr = (p.dbg & 4) && blockIdx.x == 0 && blockIdx.y == 0;
    if (tr && threadIdx.x == 0) g_ct_trace[0] = clock64();
    int mt = blockIdx.x;
    const int tx0 = (mt % tiles_x) * TW; mt /= tiles_x;
    const int ty0 = (mt % tiles_y) * TH;
    const int b = mt / tiles_y;
    const int n0 = blockIdx.y * BN;
    const int cchunks = p.cin / CT_BK;
    const int iters = p.KH * p.KW * cchunks;

    if (threadIdx.x == 0) {
        tc::prefetch_tmap(&tmA);
        tc::prefetch_tmap(&tmB);
        if (p.tma_store) tc::prefetch_tmap(&tmO);
        for (int s = 0; s < Cfg::STAGES; ++s) { tc::mbar_init(full + s, 1); tc::mbar_init(empty + s, CT_CONSUMERS); }
        if (HALO) for (int s = 0; s < HL_A_STAGES; ++s) { tc::mbar_init(a_full + s, 1); tc::mbar_init(a_empty + s, CT_CONSUMERS); }
        tc::fence_barrier_init();
    }
    __syncthreads();
    if (tr && threadIdx.x == 0) g_ct_trace[1] = clock64();

    if (warp == CT_CONSUMERS) {
        if (HALO && lane == 0) {
            int bit = 0;
            for (int cc = 0; cc < cchunks; ++cc) {
                const int a = cc % HL_A_STAGES;
                tc::mbar_wait(a_empty + a, ((cc / HL_A_STAGES) & 1) ^ 1);
                tc::mbar_arrive_expect_tx(a_full + a, HL_A_BYTES);
                tc::tma_load_4d(smem + a * HL_A_SLOT, &tmA, a_full + a, cc * CT_BK, tx0 - p.pad, ty0 - p.pad, b);
                for (int tap = 0; tap < 9; ++tap, ++bit) {
                    const int s = bit % Cfg::STAGES;
                    tc::mbar_wait(empty + s, ((bit / Cfg::STAGES) & 1) ^ 1);
                    tc::mbar_arrive_expect_tx(full + s, Cfg::B_BYTES);
                    tc::tma_load_2d(smB + s * Cfg::B_BYTES, &tmB, full + s, tap * p.cin + cc * CT_BK, n0);
                }
            }
        } else if (lane == 0) {
            for (int it = 0; it < iters; ++it) {
                const int s = it % Cfg::STAGES;
                tc::mbar_wait(empty + s, ((it / Cfg::STAGES) & 1) ^ 1);
                unsigned char* sa = smem + s * Cfg::STAGE_BYTES;
                unsigned char* sb = sa + CT_A_BYTES;
                const int tap = it / cchunks, cc = it - tap * cchunks;
                const int r = tap / p.KW, sx = tap - r * p.KW;
                const bool ldA = !(p.dbg & 2) || it < Cfg::STAGES, ldB = !(p.dbg & 1) || it < Cfg::STAGES;
                tc::mbar_arrive_expect_tx(full + s, (ldA ? CT_A_BYTES : 0) + (ldB ? Cfg::B_BYTES : 0));
                if (ldA) tc::tma_load_4d(sa, &tmA, full + s, cc * CT_BK, tx0 * p.stride + sx - p.pad, ty0 * p.stride + r - p.pad, b);
                if (ldB) tc::tma_load_2d(sb, &tmB, full + s, tap * p.cin + cc * CT_BK, n0);
            }
        }
    } else {
        // ---- main loop: warpgroup g accumulates pixels [64g, 64g+64) of the patch
        const int g = warp >> 2;
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        if (HALO) {
            int bit = 0;
            for (int cc = 0; cc < cchunks; ++cc) {
                const int a = cc % HL_A_STAGES;
                tc::mbar_wait(a_full + a, (cc / HL_A_STAGES) & 1);
                const uint32_t ha = tc::smem_u32(smem + a * HL_A_SLOT);
                for (int tap = 0; tap < 9; ++tap, ++bit) {
                    const int s = bit % Cfg::STAGES;
                    tc::mbar_wait(full + s, (bit / Cfg::STAGES) & 1);
                    const int r = tap / 3, sx = tap - r * 3;
                    // window (r, sx) of the halo for pixel rows [64g, 64g+64) = patch rows [8g, 8g+8): 8-pixel rows HL_PITCH pixels apart
                    const uint32_t a0 = ha + (uint32_t)(((r + 8 * g) * HL_PITCH + sx) * 128);
                    const uint64_t adesc = tc::smem_desc_sw128(a0, HL_PITCH * 128);
                    const uint64_t bdesc = tc::smem_desc_sw128(tc::smem_u32(smB + s * Cfg::B_BYTES));
                    tc::wgmma_fence();
#pragma unroll
                    for (int k = 0; k < CT_BK / 8; ++k)
                        tc::wgmma<BN, tc::K_TF32>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1u);
                    tc::wgmma_commit();
                    tc::wgmma_wait_one();               // this tap's MMAs stay in flight; the previous tap's weight tile is free
                    __syncwarp();
                    if (lane == 0 && bit > 0) tc::mbar_arrive(empty + (bit - 1) % Cfg::STAGES);
                    // every MMA of the previous slice has completed: its halo slot is free
                    if (lane == 0 && tap == 0 && cc > 0) tc::mbar_arrive(a_empty + (cc - 1) % HL_A_STAGES);
                }
            }
            tc::wgmma_wait_all();
        } else {
            for (int it = 0; it < iters; ++it) {
                const int s = it % Cfg::STAGES;
                if (tr && threadIdx.x == 0 && it < 20) g_ct_trace[8 + it * 2] = clock64();
                tc::mbar_wait(full + s, (it / Cfg::STAGES) & 1);
                if (tr && threadIdx.x == 0 && it < 20) g_ct_trace[9 + it * 2] = clock64();
                const uint32_t sa = tc::smem_u32(smem + s * Cfg::STAGE_BYTES);
                const uint64_t adesc = tc::smem_desc_sw128(sa + g * 64 * 128), bdesc = tc::smem_desc_sw128(sa + CT_A_BYTES);
                tc::wgmma_fence();
#pragma unroll
                for (int k = 0; k < CT_BK / 8; ++k)        // K = 8 tf32 = 32 bytes per instruction
                    tc::wgmma<BN, tc::K_TF32>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1u);
                tc::wgmma_commit();
                tc::wgmma_wait_one();                   // this step's MMAs stay in flight; the previous step's stage is free
                __syncwarp();
                if (lane == 0 && it > 0) tc::mbar_arrive(empty + (it - 1) % Cfg::STAGES);
            }
            tc::wgmma_wait_all();
        }
        // (no stage is released after the last step: the producer has nothing left to load)
        if (tr && threadIdx.x == 0) g_ct_trace[2] = clock64();
        tc::acc_to_smem<BN>(acc, acc_stg, Cfg::ACC_LD, g * 64);
        // the pipeline buffers are idle from here on: the epilogue stages its output tiles there
        tc::named_sync(1, 32 * CT_CONSUMERS);
        if (tr && threadIdx.x == 0) g_ct_trace[3] = clock64();

        // ---- epilogue: warp w handles pixels [32*(w%4), +32) and channel half w/4 of the accumulator
        const int q = warp & 3;
        const int row = q * 32 + lane;                          // pixel index inside the TH x TW patch
        constexpr int PER = BN >= 64 ? BN / 2 : BN;
        const int half = warp >> 2;
        const int y = ty0 + row / TW, x = tx0 + row % TW;
        const bool valid = (y < p.Ho) && (x < p.Wo);
        if (half == 1 && BN < 64) { /* nothing left for the second warp group */ } else
#pragma unroll 1
        for (int mc = half * PER; mc < half * PER + PER; mc += 32) {
            const int c0 = mc;
            float* orow = p.out + (((size_t)b * p.OH + (y * p.os + p.oy0)) * p.OW + (x * p.os + p.ox0)) * p.out_cstride + p.out_coff;
            float v[32];
            tc::smem_row32(acc_stg, Cfg::ACC_LD, row, mc, v);
            if (p.gmax) {
                // fused max-pool over the points of a crop (torch.max(dim=points), position_transformer.py:109,118): the 128 rows of this
                // tile belong to ONE group (gmax_rows % 128 == 0); warp-shuffle max over its 32 rows per column, one atomic per warp and
                // column.  The (rows, cout) activation is never written to HBM, the group_max pass never reads it back.
                const int grp = (p.grow0 + ty0 * p.Wo + tx0) / p.gmax_rows;
                // transpose through the (idle) pipeline buffers: row stride 33 floats => conflict-free scalar stores and column reads
                float* stg = reinterpret_cast<float*>(smem + ((mc / 32) * 4 + q) * 4352);
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const int n = n0 + c0 + j;
                    float o = v[j];
                    if (n < p.cout) {
                        if (p.scale) o *= __ldg(p.scale + n);
                        if (p.shift) o += __ldg(p.shift + n);
                        if (p.relu) o = fmaxf(o, 0.f);
                    }
                    stg[lane * 33 + j] = valid ? o : -INFINITY;
                }
                __syncwarp();
                float cm = -INFINITY;
#pragma unroll
                for (int r = 0; r < 32; ++r) cm = fmaxf(cm, stg[r * 33 + lane]);      // lane = column
                const int n = n0 + c0 + lane;
                if (n < p.cout) {
                    float* addr = p.gmax + (size_t)grp * p.cout + n;
                    if (cm >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(cm));
                    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(cm));
                }
                __syncwarp();
            } else if (p.tma_store) {
                // Per-pixel strided stores (32 lanes -> 32 different lines per instruction) would make the epilogue as long as the
                // main loop.  Here the warp's 32 pixels x 32 channels go to the (now idle) pipeline buffers in the 128B-swizzled box
                // layout and ONE TMA store per warp writes them (edge tiles clipped by the tensor map, channel range clipped at
                // out_coff + cout).  Staging slots (16 KB each, 4 KB per warp) are carved from the pipeline buffers; each warp group
                // owns half of them and a warp re-uses its 4 KB only after its own earlier TMA store has read it.
                constexpr int SLOTS_H = (Cfg::BUF / CT_A_BYTES) / 2;
                const int cj = (mc - half * PER) / 32;
                if (cj >= SLOTS_H) { if (lane == 0) tc::tma_store_wait_read(); __syncwarp(); }
                unsigned char* stg = smem + (half * SLOTS_H + cj % SLOTS_H) * CT_A_BYTES + q * 4096;        // 32 rows x 128 B
                const uint32_t stg_u = tc::smem_u32(stg) + (uint32_t)((lane >> 3) * 1024 + (lane & 7) * 128);
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                    const int n = n0 + c0 + j;
                    float4 o = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
                    if (n < p.cout) {
                        if (p.scale) { float4 sc = __ldg(reinterpret_cast<const float4*>(p.scale + n)); o.x *= sc.x; o.y *= sc.y; o.z *= sc.z; o.w *= sc.w; }
                        if (p.shift) { float4 sh = __ldg(reinterpret_cast<const float4*>(p.shift + n)); o.x += sh.x; o.y += sh.y; o.z += sh.z; o.w += sh.w; }
                        if (p.gshift && valid) {
                            float4 sh = __ldg(reinterpret_cast<const float4*>(p.gshift + (size_t)((p.grow0 + y * p.Wo + x) / p.gsize) * p.cout + n));
                            o.x += sh.x; o.y += sh.y; o.z += sh.z; o.w += sh.w;
                        }
                    }
                    if (p.relu) {
                        o.x = tc::rna_tf32(fmaxf(o.x, 0.f)); o.y = tc::rna_tf32(fmaxf(o.y, 0.f));
                        o.z = tc::rna_tf32(fmaxf(o.z, 0.f)); o.w = tc::rna_tf32(fmaxf(o.w, 0.f));
                    }
                    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(stg_u + (uint32_t)((((j >> 2) ^ (lane & 7))) << 4)),
                                 "f"(o.x), "f"(o.y), "f"(o.z), "f"(o.w) : "memory");
                }
                tc::fence_proxy_async();                 // generic-proxy smem writes -> visible to the TMA (async proxy)
                __syncwarp();
                if (lane == 0 && n0 + c0 < p.cout) {
                    const int row0 = ty0 + q * (32 / TW);      // the warp's 32 pixels = 32/TW patch rows
                    if (p.tma_store == 2) {
                        // ConvTranspose2d with kernel == stride: output pixel (y*os + oy0, x*os + ox0) through the 5-D view
                        // [C][dx][x][dy][b*Ho + y] of the NHWC tensor.  The merged (batch, y) axis cannot clip rows past Ho: skip them
                        // (Ho is even and row0 is even, so a 2-row box is either entirely inside or entirely outside)
                        if (row0 < p.Ho) tc::tma_store_5d(&tmO, stg, p.out_coff + n0 + c0, p.ox0, tx0, p.oy0, b * p.Ho + row0);
                    } else {
                        tc::tma_store_4d(&tmO, stg, p.out_coff + n0 + c0, tx0, row0, b);
                    }
                    tc::tma_store_commit();
                }
            } else if (valid) {
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                    const int n = n0 + c0 + j;
                    if (n >= p.cout) break;
                    float4 o = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
                    if (p.scale) { float4 sc = __ldg(reinterpret_cast<const float4*>(p.scale + n)); o.x *= sc.x; o.y *= sc.y; o.z *= sc.z; o.w *= sc.w; }
                    if (p.shift) { float4 sh = __ldg(reinterpret_cast<const float4*>(p.shift + n)); o.x += sh.x; o.y += sh.y; o.z += sh.z; o.w += sh.w; }
                    if (p.gshift) {
                        float4 sh = __ldg(reinterpret_cast<const float4*>(p.gshift + (size_t)((p.grow0 + y * p.Wo + x) / p.gsize) * p.cout + n));
                        o.x += sh.x; o.y += sh.y; o.z += sh.z; o.w += sh.w;
                    }
                    if (p.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
                    if (p.relu) { o.x = tc::rna_tf32(o.x); o.y = tc::rna_tf32(o.y); o.z = tc::rna_tf32(o.z); o.w = tc::rna_tf32(o.w); }  // feeds another TF32 conv
                    *reinterpret_cast<float4*>(orow + n) = o;
                }
            }
        }
        if (p.tma_store && lane == 0) tc::tma_store_wait_read();      // the stores must have read the staging buffers
    }
    if (tr && threadIdx.x == 0) g_ct_trace[4] = clock64();
}

template <int BN, bool HALO>
static int launch_tf32(const Conv2dParams& p, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, cudaStream_t st) {
    using Cfg = CtCfg<BN, HALO>;
    static bool configured = false;
    if (!configured) {
        DZ_CUDA(cudaFuncSetAttribute(k_conv2d_tf32<BN, HALO>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
        configured = true;
    }
    int tiles_x = dz_cdiv(p.Wo, Cfg::TW), tiles_y = dz_cdiv(p.Ho, Cfg::TH);
    dim3 grid(tiles_x * tiles_y * p.B, dz_cdiv(p.cout, BN));
    static_assert((BN / 32) * CT_A_BYTES <= Cfg::BUF, "epilogue staging must fit in the pipeline buffers");
    k_conv2d_tf32<BN, HALO><<<grid, CT_THREADS, Cfg::SMEM, st>>>(tmA, tmB, tmO, p, tiles_x, tiles_y);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// p.w must be in (cout, KH, KW, cin) layout for this path
int dz_conv2d_fwd_tc(const Conv2dParams& p_in, int mode, cudaStream_t st) {
    Conv2dParams p = p_in;
    if (mode != DZ_TF32) { dz_set_error("dz_conv2d_fwd: tensor-core mode %d not built (tf32 only)", mode); return DZ_ERR_UNSUPPORTED; }
    if (p.cin % CT_BK != 0 || p.in_cstride % 4 != 0 || p.cout % 4 != 0 || p.out_cstride % 4 != 0 || p.out_coff % 4 != 0) {
        dz_set_error("dz_conv2d_fwd(tf32): needs cin %% 32 == 0 and 16-byte aligned channel slices (cin=%d cout=%d)", p.cin, p.cout);
        return DZ_ERR_UNSUPPORTED;
    }
    tc::EncodeTiledFn enc = tc::get_encode_tiled();
    if (!enc) { dz_set_error("cuTensorMapEncodeTiled unavailable"); return DZ_ERR_CUDA; }
    static const int no_tma_store = getenv("DZ_CONV2D_NO_TMA_STORE") ? 1 : 0;
    p.tma_store = (!p.gmax && !no_tma_store && p.os == 1 && p.oy0 == 0 && p.ox0 == 0 && p.OH == p.Ho && p.OW == p.Wo &&
                   (reinterpret_cast<uintptr_t>(p.out) & 15) == 0) ? 1 : 0;
    // 3x3 stride-1 convolutions with at least two patches per SM and 128-channel slice: the halo variant (DZ_CONV2D_HALO=0 switches it off)
    static const int use_halo = getenv("DZ_CONV2D_HALO") ? atoi(getenv("DZ_CONV2D_HALO")) : 1;
    const long long tiles_m = (long long)dz_cdiv(p.Wo, CT_TW) * dz_cdiv(p.Ho, CT_TH) * p.B;
    const bool halo = use_halo && p.KH == 3 && p.KW == 3 && p.stride == 1 && p.tma_store == 1 && !p.gshift && !(p.dbg & 3) &&
                      tiles_m * dz_cdiv(p.cout, 128) >= 2 * DZ_NUM_SMS;
    const int TW = halo ? HL_TW : CT_TW;
    CUtensorMap tmA, tmB;
    {
        cuuint64_t dims[4] = {(cuuint64_t)p.in_cstride, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.B};
        cuuint64_t strides[3] = {(cuuint64_t)p.in_cstride * 4, (cuuint64_t)p.W * p.in_cstride * 4, (cuuint64_t)p.H * p.W * p.in_cstride * 4};
        // with a traversal stride s the box spans (n-1)*s+1 input elements and delivers n of them; the halo box is the patch + 1 pixel
        // on each side
        cuuint32_t box[4] = {(cuuint32_t)CT_BK, (cuuint32_t)((CT_TW - 1) * p.stride + 1), (cuuint32_t)((CT_TH - 1) * p.stride + 1), 1};
        if (halo) { box[1] = HL_PITCH; box[2] = HL_ROWS; }
        cuuint32_t estr[4] = {1, (cuuint32_t)p.stride, (cuuint32_t)p.stride, 1};
        CUresult r = enc(&tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)p.in, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(A) failed: %d", (int)r); return DZ_ERR_CUDA; }
    }
    const int bn = p.cout > 64 ? 128 : (p.cout > 32 ? 64 : 32);
    {
        cuuint64_t ktot = (cuuint64_t)p.KH * p.KW * p.cin;
        cuuint64_t dims[2] = {ktot, (cuuint64_t)p.cout};
        cuuint64_t strides[1] = {ktot * 4};
        cuuint32_t box[2] = {(cuuint32_t)CT_BK, (cuuint32_t)bn};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)p.w, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(B) failed: %d", (int)r); return DZ_ERR_CUDA; }
    }
    CUtensorMap tmO = tmB;
    if (!p.tma_store && !p.gmax && !no_tma_store && p.os >= 2 && p.OH == p.Ho * p.os && p.OW == p.Wo * p.os && p.Ho % 2 == 0 &&
        p.oy0 < p.os && p.ox0 < p.os && (reinterpret_cast<uintptr_t>(p.out) & 15) == 0) {
        // strided output (ConvTranspose2d as os*os 1x1 convs): 5-D view [C][dx][x][dy][b*Ho + y], one TMA store per warp as above instead of
        // per-thread strided stores
        p.tma_store = 2;
        cuuint64_t dims[5] = {(cuuint64_t)(p.out_coff + p.cout), (cuuint64_t)p.os, (cuuint64_t)p.Wo, (cuuint64_t)p.os, (cuuint64_t)p.Ho * p.B};
        cuuint64_t strides[4] = {(cuuint64_t)p.out_cstride * 4, (cuuint64_t)p.os * p.out_cstride * 4, (cuuint64_t)p.OW * p.out_cstride * 4,
                                 (cuuint64_t)p.os * p.OW * p.out_cstride * 4};
        cuuint32_t box[5] = {32, 1, (cuuint32_t)CT_TW, 1, 2};
        cuuint32_t estr[5] = {1, 1, 1, 1, 1};
        CUresult r = enc(&tmO, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, (void*)p.out, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(strided out) failed: %d", (int)r); return DZ_ERR_CUDA; }
    } else if (p.tma_store) {
        // channels [0, out_coff + cout) of the (possibly wider, concatenated) output tensor: stores past cout are clipped
        cuuint64_t dims[4] = {(cuuint64_t)(p.out_coff + p.cout), (cuuint64_t)p.OW, (cuuint64_t)p.OH, (cuuint64_t)p.B};
        cuuint64_t strides[3] = {(cuuint64_t)p.out_cstride * 4, (cuuint64_t)p.OW * p.out_cstride * 4, (cuuint64_t)p.OH * p.OW * p.out_cstride * 4};
        cuuint32_t box[4] = {32, (cuuint32_t)TW, (cuuint32_t)(32 / TW), 1};      // one warp's 32 pixels
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult r = enc(&tmO, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)p.out, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(out) failed: %d", (int)r); return DZ_ERR_CUDA; }
    }
    if (halo) switch (bn) {
        case 128: return launch_tf32<128, true>(p, tmA, tmB, tmO, st);
        case 64: return launch_tf32<64, true>(p, tmA, tmB, tmO, st);
        default: return launch_tf32<32, true>(p, tmA, tmB, tmO, st);
    }
    switch (bn) {
        case 128: return launch_tf32<128, false>(p, tmA, tmB, tmO, st);
        case 64: return launch_tf32<64, false>(p, tmA, tmB, tmO, st);
        default: return launch_tf32<32, false>(p, tmA, tmB, tmO, st);
    }
}


// y = act((x @ W^T) * scale + shift) on the tensor cores: a linear layer is a 1x1 convolution over an "image" of width 16
// whose pixels are the rows of x (an 8 x 16 patch == 128 consecutive rows), so the implicit-GEMM kernel above serves
// F.linear / Conv1d(k=1) / Conv2d(k=1) of the refiner (utils/detzero_utils/model_utils.py:81-134) unchanged.
// Requirements: K % 32 == 0, N % 4 == 0, ldy % 4 == 0; the M % 16 tail rows go through the exact-fp32 kernel.
int dz_linear_fwd_f32_rows(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift, int relu,
                           float* y, int ldy, const float* gshift, int gsize, int grow0, cudaStream_t st);

// fused Linear(+BN+ReLU) + max over groups of `group` rows -> gmax (M/group, N), pre-set to -inf by the caller.  Needs the TMA shapes
// (K % 32 == 0, N % 4 == 0) and group % 128 == 0 (a 128-row tile never straddles two groups); returns DZ_ERR_UNSUPPORTED otherwise.
int dz_linear_max_fwd_tc(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift, int relu, int group,
                         float* gmax, cudaStream_t st) {
    if (K % 32 != 0 || N % 4 != 0 || group % 128 != 0 || M % group != 0) { dz_set_error("dz_linear_max_fwd: shape not supported by the fused path"); return DZ_ERR_UNSUPPORTED; }
    const int H = M / 16;
    Conv2dParams p{x, w, scale, shift, gmax, 1, H, 16, K, K, 1, 1, 1, 0, H, 16, N, H, 16, 1, 0, 0, 0, N, relu};
    p.gmax = gmax; p.gmax_rows = group; p.grow0 = 0; p.gsize = 1;
    return dz_conv2d_fwd_tc(p, DZ_TF32, st);
}

int dz_linear_fwd_tc(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift, int relu, float* y,
                     int ldy, int mode, const float* gshift, int gsize, cudaStream_t st) {
    if (mode != DZ_TF32) { dz_set_error("dz_linear_fwd: tensor-core mode %d not built (tf32 only)", mode); return DZ_ERR_UNSUPPORTED; }
    if (K % 32 != 0 || N % 4 != 0 || ldy % 4 != 0 || M < 16)      // shapes the TMA path cannot express: exact-fp32 kernel (more precise)
        return dz_linear_fwd_f32_rows(x, M, K, w, N, scale, shift, relu, y, ldy, gshift, gsize, 0, st);
    const int H = M / 16, tail = M - H * 16;
    Conv2dParams p{x, w, scale, shift, y, 1, H, 16, K, K, 1, 1, 1, 0, H, 16, N, H, 16, 1, 0, 0, 0, ldy, relu};
    p.gshift = gshift; p.gsize = gsize > 0 ? gsize : 1; p.grow0 = 0;
    int rc = dz_conv2d_fwd_tc(p, DZ_TF32, st);
    if (rc) return rc;
    if (tail) return dz_linear_fwd_f32_rows(x + (size_t)H * 16 * K, tail, K, w, N, scale, shift, relu, y + (size_t)H * 16 * ldy, ldy, gshift, gsize, H * 16, st);
    return DZ_OK;
}

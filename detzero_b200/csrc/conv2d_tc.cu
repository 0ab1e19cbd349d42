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
// accumulators; a ring of mbarrier-guarded stages overlaps TMA with MMA.  The kernel is persistent (every resident CTA walks
// a static list of tiles) and the producer warp loads the next tile while the consumers run the epilogue straight from
// their accumulator registers: folded BatchNorm / bias / ReLU, NHWC rows written through TMA stores (optionally into a
// channel slice / strided pixels: fused torch.cat and ConvTranspose2d with kernel == stride as one GEMM), or a fused max
// over row groups.
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
static constexpr int CT_CONSUMERS = 8;                        // warps 0-7: two wgmma warpgroups, each runs its own epilogue
static constexpr int CT_THREADS = 32 * (CT_CONSUMERS + 1);    // warp 8: TMA producer
static constexpr int CT_BOX_BYTES = 16 * 128;                 // epilogue: one consumer warp's 16 pixels x 32 channels

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
    // epilogue staging, separate from the pipeline buffers (those already hold the next tile's operands): 8 warps x BN/32 boxes
    static constexpr int STG_BYTES = CT_CONSUMERS * (BN / 32) * CT_BOX_BYTES;
    static constexpr int BUDGET = 227 * 1024 - 1024 - 256 - STG_BYTES;  // H100: 227 KB of shared memory per block
    // generic: STAGES x (A patch + B tile); halo: HL_A_STAGES halo slots + STAGES B tiles
    static constexpr int STAGE_BYTES = HALO ? B_BYTES : CT_A_BYTES + B_BYTES;
    static constexpr int A_REGION = HALO ? HL_A_STAGES * HL_A_SLOT : 0;
    static constexpr int FIT = (BUDGET - A_REGION) / STAGE_BYTES;
    static constexpr int STAGES = FIT > (HALO ? 9 : 8) ? (HALO ? 9 : 8) : FIT;
    static constexpr int BUF = A_REGION + STAGES * STAGE_BYTES;         // pipeline buffers
    static constexpr int SMEM = BUF + STG_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

__device__ __forceinline__ float2 ldg2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }

// Persistent: grid = min(tiles, resident CTAs), CTA i takes tiles i, i + grid, ... (static order; a tile's accumulation order is fixed, so
// results do not depend on the grid).  Tile t = (pixel patch t / tiles_n, channel tile t % tiles_n): the channel tiles of one
// patch run back to back and re-read its activations from L2.  The producer warp runs on across tile boundaries, so the next
// tile's operands load while the consumers run the epilogue of the current one; the epilogue works straight from the wgmma
// accumulator registers and its TMA stores drain during the next tile's main loop.
template <int BN, bool HALO>
__global__ void __launch_bounds__(CT_THREADS, 1)
k_conv2d_tf32(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
              Conv2dParams p, int tiles_x, int tiles_y, int tiles_n, int tiles) {
    using Cfg = CtCfg<BN, HALO>;
    constexpr int TH = Cfg::TH, TW = Cfg::TW;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* smB = smem + Cfg::A_REGION;                              // halo: the B ring follows the halo slots
    unsigned char* stg_all = smem + Cfg::BUF;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::BUF + Cfg::STG_BYTES);
    uint64_t* empty = full + Cfg::STAGES;
    uint64_t* a_full = empty + Cfg::STAGES;                                 // halo slots
    uint64_t* a_empty = a_full + HL_A_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
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

    // ring positions (k-steps and halo slices) run on across the tiles of this CTA, in the producer and the consumers alike
    int bit = 0, hs = 0;
    if (warp == CT_CONSUMERS) {
        if (lane != 0) return;
        for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
            const int n0 = (t % tiles_n) * BN;
            int mt = t / tiles_n;
            const int tx0 = (mt % tiles_x) * TW; mt /= tiles_x;
            const int ty0 = (mt % tiles_y) * TH;
            const int b = mt / tiles_y;
            if (HALO) {
                for (int cc = 0; cc < cchunks; ++cc, ++hs) {
                    const int a = hs % HL_A_STAGES;
                    tc::mbar_wait(a_empty + a, ((hs / HL_A_STAGES) & 1) ^ 1);
                    tc::mbar_arrive_expect_tx(a_full + a, HL_A_BYTES);
                    tc::tma_load_4d(smem + a * HL_A_SLOT, &tmA, a_full + a, cc * CT_BK, tx0 - p.pad, ty0 - p.pad, b);
                    for (int tap = 0; tap < 9; ++tap, ++bit) {
                        const int s = bit % Cfg::STAGES;
                        tc::mbar_wait(empty + s, ((bit / Cfg::STAGES) & 1) ^ 1);
                        tc::mbar_arrive_expect_tx(full + s, Cfg::B_BYTES);
                        tc::tma_load_2d(smB + s * Cfg::B_BYTES, &tmB, full + s, tap * p.cin + cc * CT_BK, n0);
                    }
                }
            } else {
                for (int it = 0; it < iters; ++it, ++bit) {
                    const int s = bit % Cfg::STAGES;
                    tc::mbar_wait(empty + s, ((bit / Cfg::STAGES) & 1) ^ 1);
                    unsigned char* sa = smem + s * Cfg::STAGE_BYTES;
                    unsigned char* sb = sa + CT_A_BYTES;
                    const int tap = it / cchunks, cc = it - tap * cchunks;
                    const int r = tap / p.KW, sx = tap - r * p.KW;
                    tc::mbar_arrive_expect_tx(full + s, CT_A_BYTES + Cfg::B_BYTES);
                    tc::tma_load_4d(sa, &tmA, full + s, cc * CT_BK, tx0 * p.stride + sx - p.pad, ty0 * p.stride + r - p.pad, b);
                    tc::tma_load_2d(sb, &tmB, full + s, tap * p.cin + cc * CT_BK, n0);
                }
            }
        }
        return;
    }

    // ---- consumers: warpgroup g accumulates pixels [64g, 64g+64) of the patch; fragment row r of this thread is tile row
    // 16 * warp + lane / 4 + 8 r, its columns are 8 j + 2 (lane % 4) + {0, 1} (tc.cuh)
    const int g = warp >> 2;
    const int N = p.cout * p.os * p.os;          // GEMM columns: os x os sub-pixel groups of cout channels (ConvTranspose2d, kernel == stride)
    unsigned char* stg = stg_all + warp * (BN / 32) * CT_BOX_BYTES;      // this warp's BN/32 staging boxes (16 rows x 128 B each)
    float acc[BN / 2];
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int n0 = (t % tiles_n) * BN;
        int mt = t / tiles_n;
        const int tx0 = (mt % tiles_x) * TW; mt /= tiles_x;
        const int ty0 = (mt % tiles_y) * TH;
        const int b = mt / tiles_y;
        // this thread's per-column scale / shift, loaded before the main loop so that the epilogue does not wait for them
        float2 scl[BN / 8], shf[BN / 8];
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int n = n0 + 8 * j + 2 * (lane & 3);
            const int c = p.os == 1 ? n : n % p.cout;                  // n, n + 1 share the sub-pixel group: cout % 4 == 0
            scl[j] = (n < N && p.scale) ? ldg2(p.scale + c) : make_float2(1.f, 1.f);
            shf[j] = (n < N && p.shift) ? ldg2(p.shift + c) : make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        if (HALO) {
            for (int cc = 0; cc < cchunks; ++cc, ++hs) {
                const int a = hs % HL_A_STAGES;
                tc::mbar_wait(a_full + a, (hs / HL_A_STAGES) & 1);
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
                    if (lane == 0 && (cc > 0 || tap > 0)) tc::mbar_arrive(empty + (bit - 1) % Cfg::STAGES);
                    // every MMA of the previous slice has completed: its halo slot is free
                    if (lane == 0 && tap == 0 && cc > 0) tc::mbar_arrive(a_empty + (hs - 1) % HL_A_STAGES);
                }
            }
            tc::wgmma_wait_all();
            if (lane == 0) { tc::mbar_arrive(empty + (bit - 1) % Cfg::STAGES); tc::mbar_arrive(a_empty + (hs - 1) % HL_A_STAGES); }
        } else {
            for (int it = 0; it < iters; ++it, ++bit) {
                const int s = bit % Cfg::STAGES;
                tc::mbar_wait(full + s, (bit / Cfg::STAGES) & 1);
                const uint32_t sa = tc::smem_u32(smem + s * Cfg::STAGE_BYTES);
                const uint64_t adesc = tc::smem_desc_sw128(sa + g * 64 * 128), bdesc = tc::smem_desc_sw128(sa + CT_A_BYTES);
                tc::wgmma_fence();
#pragma unroll
                for (int k = 0; k < CT_BK / 8; ++k)        // K = 8 tf32 = 32 bytes per instruction
                    tc::wgmma<BN, tc::K_TF32>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1u);
                tc::wgmma_commit();
                tc::wgmma_wait_one();                   // this step's MMAs stay in flight; the previous step's stage is free
                __syncwarp();
                if (lane == 0 && it > 0) tc::mbar_arrive(empty + (bit - 1) % Cfg::STAGES);
            }
            tc::wgmma_wait_all();
            if (lane == 0) tc::mbar_arrive(empty + (bit - 1) % Cfg::STAGES);
        }

        // ---- epilogue from the accumulator registers: folded BatchNorm / bias / group shift / ReLU (separately rounded multiply
        // and add), then the warp's 16 pixels through its staging boxes and TMA stores, a fused max over row groups, or per-thread
        // stores
        if (p.tma_store) {                            // this warp's previous TMA stores must have read its staging boxes
            if (lane == 0) tc::tma_store_wait_read();
            __syncwarp();
        }
        const uint32_t stg_u = tc::smem_u32(stg);
        // staging element (row q = lane / 4 + 8 r, columns 8 j + 2 (lane % 4) + {0, 1}): box j / 4, 128-byte swizzle (16-byte
        // chunk k of row q sits at chunk k ^ (q % 8))
        auto stg_addr = [&](int j, int r) {
            const int q = (lane >> 2) + 8 * r, k16 = 2 * (j & 3) + ((lane & 3) >> 1);
            return stg_u + (uint32_t)((j >> 2) * CT_BOX_BYTES + q * 128 + ((k16 ^ (q & 7)) << 4) + (lane & 1) * 8);
        };
        if (p.tma_store && !p.gshift) {
            // the BEV / head convolutions: nothing but arithmetic and shared-memory stores
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    float ox = __fmul_rn(acc[4 * j + 2 * r], scl[j].x), oy = __fmul_rn(acc[4 * j + 2 * r + 1], scl[j].y);
                    if (p.shift) { ox = __fadd_rn(ox, shf[j].x); oy = __fadd_rn(oy, shf[j].y); }
                    if (p.relu) { ox = tc::rna_tf32(fmaxf(ox, 0.f)); oy = tc::rna_tf32(fmaxf(oy, 0.f)); }   // feeds another TF32 conv
                    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stg_addr(j, r)), "f"(ox), "f"(oy) : "memory");
                }
        } else {
            int ys[2], xs[2];
            bool valid[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int m = 16 * warp + (lane >> 2) + 8 * r;
                ys[r] = ty0 + m / TW; xs[r] = tx0 + m % TW;
                valid[r] = ys[r] < p.Ho && xs[r] < p.Wo;
            }
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int n = n0 + 8 * j + 2 * (lane & 3);
                const int grp = p.os == 1 ? 0 : n / p.cout;               // sub-pixel (dy, dx) of a strided output
                const int c = n - grp * p.cout;                            // output channel
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    float2 o = make_float2(__fmul_rn(acc[4 * j + 2 * r], scl[j].x), __fmul_rn(acc[4 * j + 2 * r + 1], scl[j].y));
                    if (p.shift) { o.x = __fadd_rn(o.x, shf[j].x); o.y = __fadd_rn(o.y, shf[j].y); }
                    if (p.gshift && valid[r] && n < N) {
                        const float2 gs = ldg2(p.gshift + (size_t)((p.grow0 + ys[r] * p.Wo + xs[r]) / p.gsize) * p.cout + c);
                        o.x = __fadd_rn(o.x, gs.x); o.y = __fadd_rn(o.y, gs.y);
                    }
                    if (p.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
                    if (p.gmax) {
                        // max over this thread's two rows (rows past the image do not count), kept in acc for the reduction below
                        if (!valid[r]) o = make_float2(-INFINITY, -INFINITY);
                        if (r == 0) { acc[4 * j] = o.x; acc[4 * j + 1] = o.y; }
                        else { acc[4 * j] = fmaxf(acc[4 * j], o.x); acc[4 * j + 1] = fmaxf(acc[4 * j + 1], o.y); }
                        continue;
                    }
                    if (p.relu) { o.x = tc::rna_tf32(o.x); o.y = tc::rna_tf32(o.y); }
                    if (p.tma_store) {
                        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stg_addr(j, r)), "f"(o.x), "f"(o.y) : "memory");
                    } else if (valid[r] && n < N) {
                        const int dy = grp / p.os, dx = grp - dy * p.os;
                        float* orow = p.out + (((size_t)b * p.OH + (ys[r] * p.os + dy)) * p.OW + (xs[r] * p.os + dx)) * p.out_cstride + p.out_coff;
                        *reinterpret_cast<float2*>(orow + c) = o;
                    }
                }
            }
        }
        if (p.gmax) {
            // fused max-pool over the points of a crop (torch.max(dim=points), position_transformer.py:109,118): the 128 rows of this
            // tile belong to ONE group (gmax_rows % 128 == 0).  Shuffle max over the warp's 16 rows, a max over the 8 warps through
            // shared memory, one atomic per column and tile.  The (rows, cout) activation is never written to HBM.
            float* red = reinterpret_cast<float*>(stg_all);                 // [8 warps][BN]
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    float v = acc[4 * j + c];
                    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
                    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 8));
                    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 16));
                    if (lane < 4) red[warp * BN + 8 * j + 2 * lane + c] = v;
                }
            }
            tc::named_sync(1, 32 * CT_CONSUMERS);
            if (threadIdx.x < BN && n0 + (int)threadIdx.x < N) {
                float cm = red[threadIdx.x];
#pragma unroll
                for (int w = 1; w < CT_CONSUMERS; ++w) cm = fmaxf(cm, red[w * BN + threadIdx.x]);
                const int grp = (p.grow0 + ty0 * p.Wo + tx0) / p.gmax_rows;
                float* addr = p.gmax + (size_t)grp * p.cout + n0 + threadIdx.x;
                if (__float_as_int(cm) >= 0) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(cm));      // sign bit: -0.0 takes atomicMin
                else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(cm));
            }
            tc::named_sync(1, 32 * CT_CONSUMERS);                            // red is rewritten by the next tile
        } else if (p.tma_store) {
            tc::fence_proxy_async();                 // generic-proxy smem writes -> visible to the TMA (async proxy)
            __syncwarp();
            if (lane == 0) {
#pragma unroll 1
                for (int cj = 0; cj < BN / 32; ++cj) {
                    const int n = n0 + 32 * cj;
                    if (n >= N) break;
                    if (p.tma_store == 2) {
                        // ConvTranspose2d with kernel == stride: output pixel (y*os + dy, x*os + dx) through the 5-D view
                        // [C][dx][x][dy][b*Ho + y] of the NHWC tensor; the warp's 16 pixels are one patch row (TW == 16).  The merged
                        // (batch, y) axis cannot clip rows past Ho: skip them
                        const int grp = n / p.cout, dy = grp / p.os, y = ty0 + warp;
                        if (y < p.Ho) tc::tma_store_5d(&tmO, stg + cj * CT_BOX_BYTES, p.out_coff + n - grp * p.cout, grp - dy * p.os, tx0, dy, b * p.Ho + y);
                    } else {
                        tc::tma_store_4d(&tmO, stg + cj * CT_BOX_BYTES, p.out_coff + n, tx0, ty0 + warp * (16 / TW), b);
                    }
                }
                tc::tma_store_commit();
            }
        }
    }
    if (p.tma_store && lane == 0) tc::tma_store_wait_read();      // the stores must have read the staging buffers
}

template <int BN, bool HALO>
static int launch_tf32(const Conv2dParams& p, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, cudaStream_t st) {
    using Cfg = CtCfg<BN, HALO>;
    static int ctas_per_sm = 0;                   // the small configurations fit two CTAs per SM
    if (!ctas_per_sm) {
        DZ_CUDA(cudaFuncSetAttribute(k_conv2d_tf32<BN, HALO>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
        DZ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, k_conv2d_tf32<BN, HALO>, CT_THREADS, Cfg::SMEM));
        if (ctas_per_sm < 1) ctas_per_sm = 1;
    }
    static_assert(CT_CONSUMERS * BN * 4 <= Cfg::STG_BYTES, "the group-max reduction must fit in the staging area");
    const int tiles_x = dz_cdiv(p.Wo, Cfg::TW), tiles_y = dz_cdiv(p.Ho, Cfg::TH), tiles_n = dz_cdiv(p.cout * p.os * p.os, BN);
    const long long tiles = (long long)tiles_x * tiles_y * p.B * tiles_n;
    if (tiles > INT32_MAX) { dz_set_error("dz_conv2d_fwd(tf32): %lld tiles", tiles); return DZ_ERR_UNSUPPORTED; }
    const int grid = (int)(tiles < (long long)DZ_NUM_SMS * ctas_per_sm ? tiles : (long long)DZ_NUM_SMS * ctas_per_sm);
    k_conv2d_tf32<BN, HALO><<<grid, CT_THREADS, Cfg::SMEM, st>>>(tmA, tmB, tmO, p, tiles_x, tiles_y, tiles_n, (int)tiles);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// HALO N=256 variant (the 3x3 stride-1 BEV / head convolutions with cout >= 64 and enough tiles to fill the machine): output
// channels are the wgmma M side and 256 pixels the N side, the widest instruction wgmma has (m64n256k8).  Per instruction it reads
// 2 KB of weights + 8 KB of activations for 262144 FLOP, against 2 KB + 4 KB for 131072 FLOP with the pixels on M, and every weight
// tile is reused over twice the pixels: by a model of shared-memory reads plus TMA writes per MMA clock, the traffic falls from about
// 1.0 to 0.8 of what the tensor cores need (measured on the BEV shapes: 10-30 % faster than the 128-pixel kernel).  A is the weight tile
// W[cout][(tap, cin)] as loaded for the kernel above; B is the halo of a 32 x 8 output patch, (32+2) x (8+2) pixels per 32-channel
// slice: its 32 core groups of 8 pixels are the 32 patch rows, SBO = the halo pitch, and the nine taps are nine shifted B descriptors
// into it, exactly as the A descriptors of the 128-pixel halo kernel.  BM = 128: the two consumer warpgroups take 64 channels each of
// one 32 x 8 patch.  BM = 64 (cout <= 64): a 32 x 16 patch, the warpgroups take its two 8-pixel column halves with the same 64
// weight rows (two CTAs per SM with one warpgroup each cannot fit two halo slots and a weight ring in half the shared memory).
// Per output the accumulation order (slice, tap, k8 step) is that of the kernels above, so results are bit-identical.
static constexpr int H2_TH = 32, H2_ROWS = H2_TH + 2;
static constexpr int H2_PIECE_PX = 32;                         // epilogue piece: 4 patch rows x 8 pixels
static constexpr int H2_PIECE_BYTES = H2_PIECE_PX * 128;       // x 32 channels
static constexpr int H2_STG_BYTES = 4 * 2 * H2_PIECE_BYTES;    // 4 warp pairs x 2 pieces in flight

template <int BM>
struct H2Cfg {
    static constexpr int TW = BM == 128 ? 8 : 16, PITCH = TW + 2;
    static constexpr int A_BYTES = H2_ROWS * PITCH * 128;            // halo tile delivered by the TMA unit
    static constexpr int A_SLOT = (A_BYTES + 1023) / 1024 * 1024;
    static constexpr int W_BYTES = BM * CT_BK * 4;                    // weight tile of one (tap, slice)
    static constexpr int BUDGET = 227 * 1024 - 1024 - 256 - H2_STG_BYTES - HL_A_STAGES * A_SLOT;
    static constexpr int STAGES = BUDGET / W_BYTES > 9 ? 9 : BUDGET / W_BYTES;
    static constexpr int SMEM = HL_A_STAGES * A_SLOT + STAGES * W_BYTES + H2_STG_BYTES + 1024 + 256;
};

// Persistent with the static tile order of k_conv2d_tf32: tile t = (patch t / tiles_n, channel tile t % tiles_n).
template <int BM>
__global__ void __launch_bounds__(CT_THREADS, 1)
k_conv2d_tf32_halo_n256(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmO,
                        Conv2dParams p, int tiles_x, int tiles_y, int tiles_n, int tiles) {
    using Cfg = H2Cfg<BM>;
    constexpr int TW = Cfg::TW;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* smW = smem + HL_A_STAGES * Cfg::A_SLOT;
    unsigned char* stg_all = smW + Cfg::STAGES * Cfg::W_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(stg_all + H2_STG_BYTES);
    uint64_t* empty = full + Cfg::STAGES;
    uint64_t* a_full = empty + Cfg::STAGES;
    uint64_t* a_empty = a_full + HL_A_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cchunks = p.cin / CT_BK;

    if (threadIdx.x == 0) {
        tc::prefetch_tmap(&tmA);
        tc::prefetch_tmap(&tmW);
        tc::prefetch_tmap(&tmO);
        for (int s = 0; s < Cfg::STAGES; ++s) { tc::mbar_init(full + s, 1); tc::mbar_init(empty + s, CT_CONSUMERS); }
        for (int s = 0; s < HL_A_STAGES; ++s) { tc::mbar_init(a_full + s, 1); tc::mbar_init(a_empty + s, CT_CONSUMERS); }
        tc::fence_barrier_init();
    }
    __syncthreads();

    int bit = 0, hs = 0;
    if (warp == CT_CONSUMERS) {
        if (lane != 0) return;
        for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
            const int n0 = (t % tiles_n) * BM;
            int mt = t / tiles_n;
            const int tx0 = (mt % tiles_x) * TW; mt /= tiles_x;
            const int ty0 = (mt % tiles_y) * H2_TH;
            const int b = mt / tiles_y;
            for (int cc = 0; cc < cchunks; ++cc, ++hs) {
                const int a = hs % HL_A_STAGES;
                tc::mbar_wait(a_empty + a, ((hs / HL_A_STAGES) & 1) ^ 1);
                tc::mbar_arrive_expect_tx(a_full + a, Cfg::A_BYTES);
                tc::tma_load_4d(smem + a * Cfg::A_SLOT, &tmA, a_full + a, cc * CT_BK, tx0 - p.pad, ty0 - p.pad, b);
                for (int tap = 0; tap < 9; ++tap, ++bit) {
                    const int s = bit % Cfg::STAGES;
                    tc::mbar_wait(empty + s, ((bit / Cfg::STAGES) & 1) ^ 1);
                    tc::mbar_arrive_expect_tx(full + s, Cfg::W_BYTES);
                    tc::tma_load_2d(smW + s * Cfg::W_BYTES, &tmW, full + s, tap * p.cin + cc * CT_BK, n0);
                }
            }
        }
        return;
    }

    // ---- consumers: warpgroup g accumulates weight rows [cg, cg + 64) of the tile against patch columns [xg, xg + 8); fragment row
    // r of this thread is channel cg + 16 (warp % 4) + lane / 4 + 8 r, its columns j = patch row, 2 (lane % 4) + {0, 1} = pixel of it
    const int g = warp >> 2, wq = warp & 3;
    const int cg = BM == 128 ? 64 * g : 0, xg = BM == 128 ? 0 : 8 * g;
    // epilogue: warps 2k, 2k + 1 (a pair) stage 32 channels x 32 pixels per piece, the pair's first lane stores it
    const int pair = warp >> 1;
    const bool store_lane = (warp & 1) == 0 && lane == 0;
    unsigned char* stg = stg_all + pair * 2 * H2_PIECE_BYTES;
    const int cq = 16 * (warp & 1) + (lane >> 2);              // channel within the pair's 32 (+ 8 r)
    float acc[128];
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int n0 = (t % tiles_n) * BM;
        int mt = t / tiles_n;
        const int tx0 = (mt % tiles_x) * TW; mt /= tiles_x;
        const int ty0 = (mt % tiles_y) * H2_TH;
        const int b = mt / tiles_y;
        float scl[2], shf[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int c = n0 + cg + 16 * wq + (lane >> 2) + 8 * r;
            scl[r] = (c < p.cout && p.scale) ? __ldg(p.scale + c) : 1.f;
            shf[r] = (c < p.cout && p.shift) ? __ldg(p.shift + c) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 128; ++i) acc[i] = 0.f;
        for (int cc = 0; cc < cchunks; ++cc, ++hs) {
            const int a = hs % HL_A_STAGES;
            tc::mbar_wait(a_full + a, (hs / HL_A_STAGES) & 1);
            const uint32_t ha = tc::smem_u32(smem + a * Cfg::A_SLOT);
            for (int tap = 0; tap < 9; ++tap, ++bit) {
                const int s = bit % Cfg::STAGES;
                tc::mbar_wait(full + s, (bit / Cfg::STAGES) & 1);
                const int r = tap / 3, sx = tap - r * 3;
                // window (r, sx) of the halo: patch row i = halo row r + i, columns [xg + sx, xg + sx + 8)
                const uint64_t bdesc = tc::smem_desc_sw128(ha + (uint32_t)((r * Cfg::PITCH + sx + xg) * 128), Cfg::PITCH * 128);
                const uint64_t adesc = tc::smem_desc_sw128(tc::smem_u32(smW + s * Cfg::W_BYTES) + cg * 128);
                tc::wgmma_fence();
#pragma unroll
                for (int k = 0; k < CT_BK / 8; ++k)
                    tc::wgmma<256, tc::K_TF32>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1u);
                tc::wgmma_commit();
                tc::wgmma_wait_one();
                __syncwarp();
                if (lane == 0 && (cc > 0 || tap > 0)) tc::mbar_arrive(empty + (bit - 1) % Cfg::STAGES);
                if (lane == 0 && tap == 0 && cc > 0) tc::mbar_arrive(a_empty + (hs - 1) % HL_A_STAGES);
            }
        }
        tc::wgmma_wait_all();
        if (lane == 0) { tc::mbar_arrive(empty + (bit - 1) % Cfg::STAGES); tc::mbar_arrive(a_empty + (hs - 1) % HL_A_STAGES); }

        // ---- epilogue: folded BatchNorm / bias / ReLU (separately rounded multiply and add), transposed into NHWC pieces of 4 patch rows
        // (staging row = pixel 8 (j % 4) + x, 32 channels, 128-byte swizzle), double-buffered per warp pair: before a piece is
        // published the store lane waits until every earlier store has read its buffer, so the piece after it may reuse that buffer
        const int c_pair = n0 + cg + 32 * (wq >> 1);
        const uint32_t stg_u = tc::smem_u32(stg);
#pragma unroll
        for (int k = 0; k < H2_TH / 4; ++k) {
            const uint32_t buf = stg_u + (uint32_t)((k & 1) * H2_PIECE_BYTES);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                const int j = 4 * k + jj;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int q = cq + 8 * r;
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        float o = __fmul_rn(acc[4 * j + 2 * r + c], scl[r]);
                        if (p.shift) o = __fadd_rn(o, shf[r]);
                        if (p.relu) o = tc::rna_tf32(fmaxf(o, 0.f));      // feeds another TF32 conv
                        const int pp = 8 * jj + 2 * (lane & 3) + c;
                        asm volatile("st.shared.f32 [%0], %1;" ::"r"(buf + (uint32_t)(pp * 128 + (((q >> 2) ^ (pp & 7)) << 4) + (q & 3) * 4)), "f"(o)
                                     : "memory");
                    }
                }
            }
            tc::fence_proxy_async();
            if (store_lane) tc::tma_store_wait_read();
            tc::named_sync(2 + pair, 64);
            if (store_lane && c_pair < p.cout) {
                tc::tma_store_4d(&tmO, stg + (k & 1) * H2_PIECE_BYTES, p.out_coff + c_pair, tx0 + xg, ty0 + 4 * k, b);
                tc::tma_store_commit();
            }
        }
    }
    if (store_lane) tc::tma_store_wait_read();
}

template <int BM>
static int launch_halo_n256(const Conv2dParams& p, const CUtensorMap& tmA, const CUtensorMap& tmW, const CUtensorMap& tmO, int tiles,
                            cudaStream_t st) {
    using Cfg = H2Cfg<BM>;
    static bool attr = false;
    if (!attr) {
        DZ_CUDA(cudaFuncSetAttribute(k_conv2d_tf32_halo_n256<BM>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
        attr = true;
    }
    const int tiles_x = dz_cdiv(p.Wo, Cfg::TW), tiles_y = dz_cdiv(p.Ho, H2_TH), tiles_n = dz_cdiv(p.cout, BM);
    const int grid = tiles < DZ_NUM_SMS ? tiles : DZ_NUM_SMS;
    k_conv2d_tf32_halo_n256<BM><<<grid, CT_THREADS, Cfg::SMEM, st>>>(tmA, tmW, tmO, p, tiles_x, tiles_y, tiles_n, tiles);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// p.w must be in (cout, KH, KW, cin) layout for this path.  p.os >= 2 (oy0 = ox0 = 0, KH = KW = 1) is a ConvTranspose2d with
// kernel == stride as ONE GEMM over the input pixels: N = os * os * cout columns, weights in (dy, dx, cout, cin) layout; column
// n goes to channel n % cout of output pixel (y * os + dy, x * os + dx), (dy, dx) = (n / cout) / os, % os.
int dz_conv2d_fwd_tc(const Conv2dParams& p_in, int mode, cudaStream_t st) {
    Conv2dParams p = p_in;
    if (mode != DZ_TF32) { dz_set_error("dz_conv2d_fwd: tensor-core mode %d not built (tf32 only)", mode); return DZ_ERR_UNSUPPORTED; }
    if (p.cin % CT_BK != 0 || p.in_cstride % 4 != 0 || p.cout % 4 != 0 || p.out_cstride % 4 != 0 || p.out_coff % 4 != 0) {
        dz_set_error("dz_conv2d_fwd(tf32): needs cin %% 32 == 0 and 16-byte aligned channel slices (cin=%d cout=%d)", p.cin, p.cout);
        return DZ_ERR_UNSUPPORTED;
    }
    if (p.oy0 != 0 || p.ox0 != 0 || p.OH != p.Ho * p.os || p.OW != p.Wo * p.os || (p.os > 1 && (p.KH != 1 || p.KW != 1 || p.gmax))) {
        dz_set_error("dz_conv2d_fwd(tf32): unsupported output geometry (os=%d)", p.os);
        return DZ_ERR_UNSUPPORTED;
    }
    tc::EncodeTiledFn enc = tc::get_encode_tiled();
    if (!enc) { dz_set_error("cuTensorMapEncodeTiled unavailable"); return DZ_ERR_CUDA; }
    const bool aligned = (reinterpret_cast<uintptr_t>(p.out) & 15) == 0;
    // TMA-store epilogue unless the output pointer is misaligned or a 32-channel store box would straddle two sub-pixels
    p.tma_store = (p.gmax || !aligned) ? 0 : p.os == 1 ? 1 : (p.cout % 32 == 0 ? 2 : 0);
    const int N = p.cout * p.os * p.os;
    const int bn = N > 64 ? 128 : (N > 32 ? 64 : 32);
    // 3x3 stride-1 convolutions: the N=256 halo variant for cout >= 64 when its tiles fill the machine, else the 128-pixel halo variant
    // with at least two patches per SM and 128-channel slice
    const bool halo3x3 = p.KH == 3 && p.KW == 3 && p.stride == 1 && p.tma_store == 1 && !p.gshift;
    const int bm = p.cout > 64 ? 128 : 64;
    const int h2_tw = bm == 128 ? H2Cfg<128>::TW : H2Cfg<64>::TW;
    const long long tiles_h2 = (long long)dz_cdiv(p.Wo, h2_tw) * dz_cdiv(p.Ho, H2_TH) * p.B * dz_cdiv(p.cout, bm);
    const bool halo_n256 = halo3x3 && p.cout >= 64 && tiles_h2 >= DZ_NUM_SMS;
    if (halo_n256 && tiles_h2 > INT32_MAX) { dz_set_error("dz_conv2d_fwd(tf32): %lld tiles", tiles_h2); return DZ_ERR_UNSUPPORTED; }
    const long long tiles_m = (long long)dz_cdiv(p.Wo, CT_TW) * dz_cdiv(p.Ho, CT_TH) * p.B;
    const bool halo = !halo_n256 && halo3x3 && tiles_m * dz_cdiv(p.cout, 128) >= 2 * DZ_NUM_SMS;
    const int TW = halo ? HL_TW : CT_TW;
    CUtensorMap tmA, tmB;
    {
        cuuint64_t dims[4] = {(cuuint64_t)p.in_cstride, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.B};
        cuuint64_t strides[3] = {(cuuint64_t)p.in_cstride * 4, (cuuint64_t)p.W * p.in_cstride * 4, (cuuint64_t)p.H * p.W * p.in_cstride * 4};
        // with a traversal stride s the box spans (n-1)*s+1 input elements and delivers n of them; the halo box is the patch + 1 pixel
        // on each side
        cuuint32_t box[4] = {(cuuint32_t)CT_BK, (cuuint32_t)((CT_TW - 1) * p.stride + 1), (cuuint32_t)((CT_TH - 1) * p.stride + 1), 1};
        if (halo) { box[1] = HL_PITCH; box[2] = HL_ROWS; }
        if (halo_n256) { box[1] = h2_tw + 2; box[2] = H2_ROWS; }
        cuuint32_t estr[4] = {1, (cuuint32_t)p.stride, (cuuint32_t)p.stride, 1};
        CUresult r = enc(&tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)p.in, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(A) failed: %d", (int)r); return DZ_ERR_CUDA; }
    }
    {
        cuuint64_t ktot = (cuuint64_t)p.KH * p.KW * p.cin;
        cuuint64_t dims[2] = {ktot, (cuuint64_t)N};
        cuuint64_t strides[1] = {ktot * 4};
        cuuint32_t box[2] = {(cuuint32_t)CT_BK, (cuuint32_t)bn};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)p.w, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(B) failed: %d", (int)r); return DZ_ERR_CUDA; }
    }
    CUtensorMap tmO = tmB;
    if (p.tma_store == 2) {
        // strided output: 5-D view [C][dx][x][dy][b*Ho + y] of the NHWC tensor, box = one warp's 16 pixels (one patch row) x 32 channels
        cuuint64_t dims[5] = {(cuuint64_t)(p.out_coff + p.cout), (cuuint64_t)p.os, (cuuint64_t)p.Wo, (cuuint64_t)p.os, (cuuint64_t)p.Ho * p.B};
        cuuint64_t strides[4] = {(cuuint64_t)p.out_cstride * 4, (cuuint64_t)p.os * p.out_cstride * 4, (cuuint64_t)p.OW * p.out_cstride * 4,
                                 (cuuint64_t)p.os * p.OW * p.out_cstride * 4};
        cuuint32_t box[5] = {32, 1, (cuuint32_t)CT_TW, 1, 1};
        cuuint32_t estr[5] = {1, 1, 1, 1, 1};
        CUresult r = enc(&tmO, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, (void*)p.out, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(strided out) failed: %d", (int)r); return DZ_ERR_CUDA; }
    } else if (p.tma_store) {
        // channels [0, out_coff + cout) of the (possibly wider, concatenated) output tensor: stores past cout are clipped
        cuuint64_t dims[4] = {(cuuint64_t)(p.out_coff + p.cout), (cuuint64_t)p.OW, (cuuint64_t)p.OH, (cuuint64_t)p.B};
        cuuint64_t strides[3] = {(cuuint64_t)p.out_cstride * 4, (cuuint64_t)p.OW * p.out_cstride * 4, (cuuint64_t)p.OH * p.OW * p.out_cstride * 4};
        cuuint32_t box[4] = {32, (cuuint32_t)TW, (cuuint32_t)(16 / TW), 1};      // one warp's 16 pixels
        if (halo_n256) { box[1] = 8; box[2] = H2_PIECE_PX / 8; }                // one epilogue piece of a warp pair
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult r = enc(&tmO, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)p.out, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(out) failed: %d", (int)r); return DZ_ERR_CUDA; }
    }
    if (halo_n256)
        return bm == 128 ? launch_halo_n256<128>(p, tmA, tmB, tmO, (int)tiles_h2, st) : launch_halo_n256<64>(p, tmA, tmB, tmO, (int)tiles_h2, st);
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

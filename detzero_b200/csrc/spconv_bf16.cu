// spconv_bf16.cu -- persistent, warp-specialised sparse convolution forward on wgmma with bf16 operand PLANES (sm_90a).
//
// Same contract as spconv.cu / spconv_tc.cu (SubMConv3d / SparseConv3d + folded BatchNorm1d + bias + residual + ReLU,
// detection/detzero_det/models/centerpoint_modules/backbone3d.py:64-83,105-121) for the modes DZ_BF16 and DZ_BF16X2.
//
// Feature storage ("planes"): a row holds PLANES x C bf16 values, [plane 0 | plane 1].
//   PLANES = 1 (DZ_BF16)   : x ~ p0                     = RN_bf16(x)                       2 bytes / value
//   PLANES = 2 (DZ_BF16X2) : x ~ p0 + p1, p1 = RN_bf16(x - p0)  (16 significand bits)      4 bytes / value (= fp32 storage)
// Weights are split the same way (w = w0 + w1).  The products are accumulated in fp32 registers as
//   PLANES = 1:  p0 * w0
//   PLANES = 2:  p0 * w0 + p0 * w1 + p1 * w0
// i.e. x*w up to the dropped p1*w1 term and the 2^-18 representation error of each operand: per-layer error ~1e-6..1e-5
// relative to fp32 FMA (tests: <= 2e-5 per layer, <= 2e-4 through a whole backbone) at the MMA and gather cost of ONE
// TF32 pass (bf16 wgmma has K = 16 per instruction, a 128-byte smem row holds 64 channels).
//
// Kernel structure (one CTA per SM, persistent over the tile list; roles by warp):
//   warps 0-7      two consumer warpgroups (64 rows each): wgmma bf16 (M64 x Cout x K16) into register accumulators; after the
//                  tile's last block every consumer thread runs the epilogue of its own fragment (two rows, two adjacent
//                  columns per 8): scale/shift (+residual) -> ReLU -> plane split -> a 4 x 4 word transpose within each quad ->
//                  16-byte stores (32-bit at Cout = 16), with no staging tile and no barrier between the warpgroups
//   warps 8-15     producers (all of them fill one pipeline stage at a time): cp.async zero-fill gather of the neighbour rows of a 64-element block of
//                  the (offset, channel) reduction dimension into K-major SW128 smem.  A lane's arrival on the stage barrier is
//                  asynchronous (cp.async.mbarrier.arrive.noinc), so it moves on to the next free stage at once: the gathers of
//                  every free stage of the ring are in flight together, and their number grows with the stage count
//   fence warp     one thread turns "the cp.async data of stage s has landed" (async mbarrier arrival of the producers) into "stage s
//                  is visible to the tensor core": fence.proxy.async, then arrives on the barrier the consumers wait on, so
//                  neither the producers nor the consumers wait for the landing latency themselves
//   tile warp      walks the CTA's tiles (heaviest-first tile order of the rulebook schedule, serpentine over the CTAs), loads
//                  the 128 x 27 neighbour rows of tile t+1/t+2 into the double-buffered table while tile t is computed
//   weight warp    one thread TMA-loads the weight slice ([w0 ; w1] rows x 64 reduction elements) of each live block into the
//                  weight ring, in the consumers' block order
// so a tile's prologue (table load) hides under the neighbouring tile's main loop and the producers run ahead into the next
// tile while the consumers run the epilogue.  No atomics: deterministic; a row's accumulation order over
// the reduction blocks never depends on the schedule, so results are bit-identical with or without it.
//
// Shared memory (SbCfg, <= 227 KB): [A ring: STAGES x PLANES x 16 KB][weight ring: WSTAGES x PLANES x COUT x 128 B]
// [table 2 x 14 KB][block lists, scale/shift, barriers].  The gathered A block and its weight slice have separate rings: the
// weight slice only has to cover the MMA look-ahead (one block in flight, one being issued, one loading), so the rest of
// shared memory goes to A stages, i.e. to gathers in flight, and what is left after them to weight slots.  bf16x2: 5 A
// stages at Cout = 16 and 32, 4 at Cout = 64, 3 at Cout = 128; bf16: 8 at every Cout.  The weight warp keeps the
// tile's block list in registers, so it releases the table buffer as soon as it has read it, like the other roles.
#include <cuda_bf16.h>
#include "common.cuh"
#include "tc.cuh"

namespace {

constexpr int SB_ROWS = 128;
constexpr int SB_A_BYTES = SB_ROWS * 128;          // one 64-element bf16 block for 128 rows
constexpr int SB_KMAX = 27;
constexpr int SB_NPLANES = SB_KMAX + 1;             // a tile block: plane k < K = neighbour rows, plane K = the tile's output rows

template <int COUT, int PLANES>
struct SbCfg {
    static constexpr int WROWS = PLANES * COUT;                     // rows of the weight tile: [w0 ; w1]
    static constexpr int W_BYTES = WROWS * 128;
    static constexpr int STAGE_BYTES = PLANES * SB_A_BYTES;         // one gathered A block
    static constexpr int NBR_BYTES = 2 * SB_NPLANES * SB_ROWS * 4;   // double-buffered tile block: K neighbour planes + the row plane
    static constexpr int MISC_BYTES = 2 * 64 * 4 + 2 * COUT * 4 + 512;                     // block lists | scale,shift | barriers
    static constexpr int RING_BYTES = 232448 - NBR_BYTES - MISC_BYTES - 1024;               // A ring + weight ring
    // weight ring: at least one slot under the MMA still in flight, one for the MMA being issued and one loading; the A ring
    // takes as many stages as fit beside that (up to 8), and what is left deepens the weight ring (up to 8 slots)
    static constexpr int STAGES_FIT = (RING_BYTES - 3 * W_BYTES) / STAGE_BYTES;
    static constexpr int STAGES = STAGES_FIT > 8 ? 8 : STAGES_FIT;   // 3 (bf16x2, Cout = 128) .. 8
    static constexpr int WSTAGES_FIT = (RING_BYTES - STAGES * STAGE_BYTES) / W_BYTES;
    static constexpr int WSTAGES = WSTAGES_FIT > 8 ? 8 : WSTAGES_FIT;
    static_assert((3 * STAGES + 2 * WSTAGES + 4) * 8 <= 512, "barriers");
    // ALL producer warps fill ONE stage at a time (16 rows each): a stage is complete after 1/NPROD of the LSU time a
    // warp-per-stage split needs, so the oldest stage lands early and the ring covers the MMA -> commit -> refill latency
    // with the two consumer warpgroups holding Cout/2 accumulator registers each, 8 producer warps leave too few registers for
    // Cout >= 64 (spills): 4 there
    static constexpr int NPROD = COUT >= 64 ? 4 : 8;
    static constexpr int CONSUMERS = 8;
    static constexpr int WARP_TILE = CONSUMERS + NPROD;
    static constexpr int WARP_FENCE = WARP_TILE + 1;
    static constexpr int WARP_W = WARP_FENCE + 1;
    static constexpr int THREADS = 32 * (WARP_W + 1);
    static constexpr int SMEM = STAGES * STAGE_BYTES + WSTAGES * W_BYTES + NBR_BYTES + MISC_BYTES + 1024;
};

// bounded wait: a protocol bug turns into a trap (CUDA error) instead of a hung GPU
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!tc::mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 24)) __trap();          // (no printf: a call anywhere in the kernel serialises its wgmma pipeline)
    }
}
// bulk copy global -> shared, completion counted in bytes on an mbarrier
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(tc::smem_u32(smem_dst)), "l"(src), "r"(bytes), "r"(tc::smem_u32(bar)) : "memory");
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
// a[i] for a lane-dependent i, by selects (an indexed register array would go to local memory)
__device__ __forceinline__ uint32_t sel4(const uint32_t (&a)[4], int i) { return i == 0 ? a[0] : i == 1 ? a[1] : i == 2 ? a[2] : a[3]; }

template <int CIN_PAD, int COUT, int PLANES>
__global__ void __launch_bounds__(SbCfg<COUT, PLANES>::THREADS, 1)
k_spconv_bf16(const __grid_constant__ CUtensorMap tmW, const uint16_t* __restrict__ in, const int32_t* __restrict__ tab, int K, int tab_rows,
              const int32_t* __restrict__ order, const int* __restrict__ d_n_out, int out_cap, const float* __restrict__ scale,
              const float* __restrict__ shift, const uint16_t* __restrict__ residual, int relu, uint16_t* __restrict__ out,
              const int32_t* __restrict__ tab_tiles) {
    using Cfg = SbCfg<COUT, PLANES>;
    constexpr int S = Cfg::STAGES;
    const int n = min(*d_n_out, out_cap);
    const int tiles_cap = (tab_rows + SB_ROWS - 1) / SB_ROWS;            // tile_order has one entry per capacity tile
    const int tiles_n = (n + SB_ROWS - 1) / SB_ROWS;
    if ((int)blockIdx.x >= tiles_n) return;                              // more CTAs than tiles: nothing to do (uniform per CTA)

    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    constexpr int WS = Cfg::WSTAGES;
    unsigned char* s_w = smem + S * Cfg::STAGE_BYTES;                              // [WS] weight slices of the live blocks
    int* s_nbr = reinterpret_cast<int*>(s_w + WS * Cfg::W_BYTES);                 // [2][28][128]: planes k < K neighbour rows, plane K = output rows (-1: none)
    int* s_blk = s_nbr + 2 * SB_NPLANES * SB_ROWS;                                // [2][64]  live reduction blocks; [63] = count, [62] = tile (-1: end)
    float* s_scale = reinterpret_cast<float*>(s_blk + 2 * 64);
    float* s_shift = s_scale + COUT;
    uint64_t* full = reinterpret_cast<uint64_t*>(s_shift + COUT);
    uint64_t* empty = full + S;
    uint64_t* landed = empty + S;                  // producers' cp.async data of a stage have landed (generic proxy)
    uint64_t* nbr_full = landed + S;
    uint64_t* nbr_empty = nbr_full + 2;
    uint64_t* wfull = nbr_empty + 2;               // weight slot loaded (TMA bytes)
    uint64_t* wempty = wfull + WS;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ktot = K * CIN_PAD;
    const int nb_tot = (ktot + 63) / 64;

    if (threadIdx.x == 0) {
        tc::prefetch_tmap(&tmW);
        for (int s = 0; s < S; ++s) { tc::mbar_init(landed + s, 32 * Cfg::NPROD); tc::mbar_init(full + s, 1); tc::mbar_init(empty + s, Cfg::CONSUMERS); }
        for (int s = 0; s < WS; ++s) { tc::mbar_init(wfull + s, 1); tc::mbar_init(wempty + s, Cfg::CONSUMERS); }
        for (int b = 0; b < 2; ++b) {
            tc::mbar_init(nbr_full + b, 1);
            tc::mbar_init(nbr_empty + b, Cfg::NPROD + 1 + Cfg::CONSUMERS + 1);    // producers, fence warp, consumers, weight warp
        }
        tc::fence_barrier_init();
    }
    for (int c = threadIdx.x; c < COUT; c += blockDim.x) {
        s_scale[c] = scale ? __ldg(scale + c) : 1.f;
        s_shift[c] = shift ? __ldg(shift + c) : 0.f;
    }
    __syncthreads();

    if (warp == Cfg::WARP_TILE) {
        // ================= tile warp: neighbour rows + live block list of the CTA's next tile ===================================
        const int G = gridDim.x;
        int t = 0;
        for (int round = 0;; ++round) {
            const int q = round * G + ((round & 1) ? (G - 1 - (int)blockIdx.x) : (int)blockIdx.x);    // serpentine over the CTAs
            const bool end = round * G >= tiles_cap;
            int tile = -1;
            if (!end) {
                if (q >= tiles_cap) continue;
                tile = order ? __ldg(order + tab_rows + q) : q;
                if (tile * SB_ROWS >= n) continue;                       // capacity tile beyond the live rows
            }
            const int b = t & 1;
            if (t >= 2) mbar_wait_bounded(nbr_empty + b, (((t >> 1) - 1) & 1));
            int* nb_b = s_nbr + b * SB_NPLANES * SB_ROWS;
            if (end) {
                if (lane == 0) s_blk[b * 64 + 62] = -1;
                __syncwarp();
                if (lane == 0) tc::mbar_arrive(nbr_full + b);
                break;
            }
            unsigned mask = 0;
            if (tab_tiles) {
                mask = (unsigned)__ldg(order + tab_rows + tiles_cap + tile);       // precomputed OR of the tile's row masks
            } else {
#pragma unroll 1
            for (int i = 0; i < 4; ++i) {
                const int r = lane + 32 * i;
                const int pos = tile * SB_ROWS + r;
                const int src = pos < n ? (order ? __ldg(order + pos) : pos) : -1;
                int w[28];
                const int4* rowp = reinterpret_cast<const int4*>(tab) + (size_t)(src < 0 ? 0 : src) * 8;
#pragma unroll
                for (int qq = 0; qq < 7; ++qq) {
                    const int4 t4 = src >= 0 ? __ldg(rowp + qq) : make_int4(-1, -1, -1, 0);
                    w[4 * qq] = t4.x; w[4 * qq + 1] = t4.y; w[4 * qq + 2] = t4.z; w[4 * qq + 3] = t4.w;
                }
                if (src < 0) w[27] = 0;
#pragma unroll
                for (int k = 0; k < SB_KMAX; ++k)
                    if (k < K) nb_b[k * SB_ROWS + r] = w[k];
                mask |= (unsigned)w[27];
                nb_b[K * SB_ROWS + r] = src;
            }
            }
            mask = __reduce_or_sync(0xffffffffu, mask);
            // live blocks: block kb covers offsets [kb*64/CIN_PAD, (kb*64+63)/CIN_PAD]
            int cnt = 0;
            for (int kb0 = 0; kb0 < nb_tot; kb0 += 32) {
                const int kb = kb0 + lane;
                bool live = false;
                if (kb < nb_tot) {
                    const int k_lo = (kb * 64) / CIN_PAD, k_hi = min(K - 1, (kb * 64 + 63) / CIN_PAD);
                    for (int k = k_lo; k <= k_hi; ++k) live |= (mask >> k) & 1u;
                }
                const unsigned bal = __ballot_sync(0xffffffffu, live);
                if (live) s_blk[b * 64 + cnt + __popc(bal & ((1u << lane) - 1u))] = kb;
                cnt += __popc(bal);
            }
            if (lane == 0) { s_blk[b * 64 + 63] = cnt; s_blk[b * 64 + 62] = tile; }
            __syncwarp();
            if (lane == 0) {
                if (tab_tiles) {                                         // the tile's (K+1) x 128 block: ONE bulk copy, completes the phase
                    const uint32_t bytes = (uint32_t)(K + 1) * SB_ROWS * 4;
                    tc::mbar_arrive_expect_tx(nbr_full + b, bytes);
                    bulk_g2s(nb_b, tab_tiles + (size_t)tile * (K + 1) * SB_ROWS, bytes, nbr_full + b);
                } else {
                    tc::mbar_arrive(nbr_full + b);                       // release: smem writes of the warp are ordered before the arrive
                }
            }
            ++t;
        }
    } else if (warp >= Cfg::CONSUMERS && warp < Cfg::CONSUMERS + Cfg::NPROD) {
        // ================= producers ============================================================================================
        const int pw = warp - Cfg::CONSUMERS;
        constexpr int RPW = SB_ROWS / Cfg::NPROD;    // rows per producer warp (16 or 32)
        constexpr int RPL = RPW / 4;                 // rows per lane (8 lanes cover the 8 chunks of a row): 4 or 8 = one or two int4 of the table
        const int j = lane & 7, rg = lane >> 3;
        const int rbase = pw * RPW + rg * RPL;
        const uint32_t smem_u = tc::smem_u32(smem);
        int g = 0;                                   // CTA-wide step counter (same sequence in every role)
        for (int t = 0;; ++t) {
            const int b = t & 1;
            mbar_wait_bounded(nbr_full + b, (t >> 1) & 1);
            if (s_blk[b * 64 + 62] < 0) break;
            const int nb = s_blk[b * 64 + 63];
            const int* nb_b = s_nbr + b * SB_NPLANES * SB_ROWS;
            for (int i = 0; i < nb; ++i) {
                const int gi = g + i;
                const int my_s = gi % S;
                const int kb = s_blk[b * 64 + i];
                mbar_wait_bounded(empty + my_s, ((gi / S) & 1) ^ 1);
                const uint32_t sa_u = smem_u + (uint32_t)(my_s * Cfg::STAGE_BYTES);
                const int e = kb * 64 + j * 8;                       // position of this lane's chunk in the (offset, channel) dimension
                const int k = e / CIN_PAD, c = e % CIN_PAD;
                const bool k_ok = k < K;
                const int4* nb_k = reinterpret_cast<const int4*>(nb_b + (k_ok ? k : 0) * SB_ROWS + rbase);
                const uint16_t* in_c = in + c;
#pragma unroll
                for (int i0 = 0; i0 < RPL; i0 += 4) {
                    const int4 nq = nb_k[i0 / 4];
                    const int rows4[4] = {nq.x, nq.y, nq.z, nq.w};
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int src_row = k_ok ? rows4[u] : -1;
                        const bool ok = src_row >= 0;
                        const int r = rbase + i0 + u;
                        const int rr = r & 7;
                        const uint32_t dst = sa_u + (uint32_t)((r >> 3) * 1024 + rr * 128 + ((j ^ rr) << 4));
                        const uint16_t* src = ok ? in_c + (size_t)src_row * (PLANES * CIN_PAD) : in;
#pragma unroll
                        for (int p = 0; p < PLANES; ++p)
                            tc::cp_async16_zfill(dst + p * SB_A_BYTES, src + (ok ? p * CIN_PAD : 0), ok);
                    }
                }
                tc::cp_async_mbar_arrive_noinc(landed + my_s);       // asynchronous: arrives when this thread's copies have landed
            }
            g += nb;
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(nbr_empty + b);
        }
    } else if (warp == Cfg::WARP_FENCE) {
        // ================= fence warp: landed[s] -> fence.proxy.async -> full[s] ===============================================
        if (lane == 0) {
            int g = 0;
            for (int t = 0;; ++t) {
                const int b = t & 1;
                mbar_wait_bounded(nbr_full + b, (t >> 1) & 1);
                if (s_blk[b * 64 + 62] < 0) break;
                const int nb = s_blk[b * 64 + 63];
                tc::mbar_arrive(nbr_empty + b);
                for (int i = 0; i < nb; ++i, ++g) {
                    const int s = g % S;
                    mbar_wait_bounded(landed + s, (g / S) & 1);
                    tc::fence_proxy_async();            // cp.async (generic proxy) writes -> tensor-core (async proxy) reads
                    tc::mbar_arrive(full + s);
                }
            }
        }
    } else if (warp == Cfg::WARP_W) {
        // ================= weight warp: TMA of each live block's weight slice into the weight ring ===============================
        int g = 0;
        for (int t = 0;; ++t) {
            const int b = t & 1;
            mbar_wait_bounded(nbr_full + b, (t >> 1) & 1);
            if (s_blk[b * 64 + 62] < 0) break;
            const int nb = s_blk[b * 64 + 63];
            // the block list (<= 54 entries) in registers, so the table buffer is released before the weight loads wait on the ring
            const int kb_lo = s_blk[b * 64 + lane], kb_hi = s_blk[b * 64 + 32 + (lane < 30 ? lane : 0)];
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(nbr_empty + b);
            for (int i = 0; i < nb; ++i, ++g) {
                const int kb = __shfl_sync(0xffffffffu, i < 32 ? kb_lo : kb_hi, i & 31);
                if (lane == 0) {
                    const int ws = g % WS;
                    mbar_wait_bounded(wempty + ws, ((g / WS) & 1) ^ 1);
                    tc::mbar_arrive_expect_tx(wfull + ws, Cfg::W_BYTES);
                    tc::tma_load_2d(s_w + ws * Cfg::W_BYTES, &tmW, wfull + ws, kb * 64, 0);
                }
                __syncwarp();
            }
        }
    } else {
        // ================= consumers: warpgroup cg accumulates rows [64cg, 64cg+64) of each tile and runs their epilogue ========
        const int cg = warp >> 2;
        const uint32_t smem_u = tc::smem_u32(smem);
        const int frow = cg * 64 + 16 * (warp & 3) + (lane >> 2);     // tile rows frow, frow + 8 of this thread's fragment
        const int fcol = 2 * (lane & 3);                               // its columns 8j + fcol, 8j + fcol + 1
        int g = 0;
        for (int t = 0;; ++t) {
            const int b = t & 1;
            mbar_wait_bounded(nbr_full + b, (t >> 1) & 1);
            if (s_blk[b * 64 + 62] < 0) break;
            const int nb = s_blk[b * 64 + 63];
            const int* rows_b = s_nbr + b * SB_NPLANES * SB_ROWS + K * SB_ROWS;
            const int orow[2] = {rows_b[frow], rows_b[frow + 8]};
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(nbr_empty + b);
            float acc[COUT / 2];
#pragma unroll
            for (int i = 0; i < COUT / 2; ++i) acc[i] = 0.f;
            for (int i = 0; i < nb; ++i, ++g) {
                const int s = g % S, ws = g % WS;
                mbar_wait_bounded(wfull + ws, (g / WS) & 1);
                mbar_wait_bounded(full + s, (g / S) & 1);
                // (the generic->async proxy fence is executed by the fence warp before it arrives)
                const uint32_t sa = smem_u + (uint32_t)(s * Cfg::STAGE_BYTES) + cg * 64 * 128;
                const uint32_t sw = tc::smem_u32(s_w + ws * Cfg::W_BYTES);
                const uint64_t a0 = tc::smem_desc_sw128(sa), w0 = tc::smem_desc_sw128(sw);
                tc::wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) tc::wgmma<COUT, tc::K_BF16>(acc, a0 + (uint64_t)(kk * 2), w0 + (uint64_t)(kk * 2), 1u);
                if (PLANES == 2) {
                    const uint64_t a1 = tc::smem_desc_sw128(sa + SB_A_BYTES), w1 = tc::smem_desc_sw128(sw + COUT * 128);
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        tc::wgmma<COUT, tc::K_BF16>(acc, a0 + (uint64_t)(kk * 2), w1 + (uint64_t)(kk * 2), 1u);
                        tc::wgmma<COUT, tc::K_BF16>(acc, a1 + (uint64_t)(kk * 2), w0 + (uint64_t)(kk * 2), 1u);
                    }
                }
                tc::wgmma_commit();
                tc::wgmma_wait_one();                   // this step's MMAs stay in flight; the previous step's stage is free
                __syncwarp();
                if (lane == 0 && i > 0) { tc::mbar_arrive(empty + (g - 1) % S); tc::mbar_arrive(wempty + (g - 1) % WS); }
            }
            tc::wgmma_wait_all();
            __syncwarp();
            if (lane == 0 && nb > 0) { tc::mbar_arrive(empty + (g - 1) % S); tc::mbar_arrive(wempty + (g - 1) % WS); }
            // epilogue straight from the accumulator fragment (tc.cuh: d[4j + 2r + c] = D[frow + 8r][8j + fcol + c]): scale/shift
            // (+ residual plane 0, then plane 1) -> ReLU -> plane split, two adjacent columns (one 32-bit word per plane) per
            // thread.  With Cout >= 32 the quad (the 4 lanes of a row) then transposes each group of 4 column blocks, so every
            // lane stores one 16-byte vector (8 columns) per plane instead of four 32-bit words: a quarter of the store
            // instructions, each writing 64 contiguous bytes per row instead of 16.  Same words, same addresses
            constexpr int QG = COUT >= 32 ? 4 : 1;                        // column blocks per quad transpose
            const int q = lane & 3;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const bool live = orow[r] >= 0;                            // uniform over the quad, not the warp: shuffles stay outside
                const size_t rbase = (size_t)(live ? orow[r] : 0) * (PLANES * COUT);
                const uint32_t* rp = residual ? reinterpret_cast<const uint32_t*>(residual + rbase + fcol) : nullptr;
#pragma unroll
                for (int j0 = 0; j0 < COUT / 8; j0 += QG) {
                    uint32_t h[PLANES][QG];
#pragma unroll
                    for (int t = 0; t < QG; ++t) {
                        const int j = j0 + t, c = 8 * j + fcol;
                        float o0 = fmaf(acc[4 * j + 2 * r], s_scale[c], s_shift[c]);
                        float o1 = fmaf(acc[4 * j + 2 * r + 1], s_scale[c + 1], s_shift[c + 1]);
                        if (rp && live) {
#pragma unroll
                            for (int p = 0; p < PLANES; ++p) {
                                const uint32_t u = __ldg(rp + (p * COUT + 8 * j) / 2);
                                o0 += bf16_lo(u); o1 += bf16_hi(u);
                            }
                        }
                        if (relu) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); }
                        h[0][t] = pack_bf16(o0, o1);
                        if (PLANES == 2) h[1][t] = pack_bf16(o0 - bf16_lo(h[0][t]), o1 - bf16_hi(h[0][t]));
                    }
#pragma unroll
                    for (int p = 0; p < PLANES; ++p) {
                        uint32_t* op = reinterpret_cast<uint32_t*>(out + rbase + p * COUT);
                        if constexpr (QG == 1) {
                            if (live) op[4 * j0 + q] = h[p][0];
                        } else {
                        // lane q gathers column block j0 + q: in round t it takes, from lane q ^ t, that lane's word of block q
                        uint32_t v[4];
#pragma unroll
                        for (int t = 0; t < 4; ++t) {
                            const uint32_t send = sel4(h[p], q ^ t);          // the block the partner lane q ^ t needs from me
                            v[t] = t ? __shfl_xor_sync(0xffffffffu, send, t) : send;
                        }
                        // word s of the vector (columns 2s, 2s+1 of the block) came from lane s, i.e. in round q ^ s
                        const uint4 w = make_uint4(sel4(v, q), sel4(v, q ^ 1), sel4(v, q ^ 2), sel4(v, q ^ 3));
                        if (live) *reinterpret_cast<uint4*>(op + 4 * (j0 + q)) = w;
                        }
                    }
                }
            }
        }
    }
}

// ---- tensor-map cache: the weight matrix of a layer never moves, encode its map once ---------------------------------------
struct TmKey { const void* p; int rows, ktot; };
struct TmEnt { TmKey k; CUtensorMap m; };
static TmEnt g_tm[128];
static int g_tm_n = 0;

static const CUtensorMap* weight_map(const void* w, int rows, int ktot) {
    for (int i = 0; i < g_tm_n; ++i)
        if (g_tm[i].k.p == w && g_tm[i].k.rows == rows && g_tm[i].k.ktot == ktot) return &g_tm[i].m;
    tc::EncodeTiledFn enc = tc::get_encode_tiled();
    if (!enc) { dz_set_error("cuTensorMapEncodeTiled unavailable"); return nullptr; }
    static CUtensorMap scratch;
    CUtensorMap* m = g_tm_n < 128 ? &g_tm[g_tm_n].m : &scratch;
    cuuint64_t dims[2] = {(cuuint64_t)ktot, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ktot * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(W bf16) failed: %d", (int)r); return nullptr; }
    if (g_tm_n < 128) { g_tm[g_tm_n].k = TmKey{w, rows, ktot}; ++g_tm_n; }
    return m;
}

template <int CIN_PAD, int COUT, int PLANES>
int launch(const void* in, const int32_t* tab, int K, int tab_rows, const int32_t* order, const int* d_n_out, int out_cap, const void* weight,
           const float* scale, const float* shift, const void* residual, int relu, void* out, const int32_t* tab_tiles, cudaStream_t st) {
    using Cfg = SbCfg<COUT, PLANES>;
    static_assert(Cfg::SMEM <= 232448, "shared memory budget");
    static bool configured = false;
    if (!configured) {
        DZ_CUDA(cudaFuncSetAttribute(k_spconv_bf16<CIN_PAD, COUT, PLANES>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
        configured = true;
    }
    const CUtensorMap* tm = weight_map(weight, Cfg::WROWS, K * CIN_PAD);
    if (!tm) return DZ_ERR_CUDA;
    const int grid = min(DZ_NUM_SMS, dz_cdiv(out_cap, SB_ROWS));
    k_spconv_bf16<CIN_PAD, COUT, PLANES><<<grid, Cfg::THREADS, Cfg::SMEM, st>>>(
        *tm, (const uint16_t*)in, tab, K, tab_rows, order, d_n_out, out_cap, scale, shift, (const uint16_t*)residual, relu, (uint16_t*)out,
        order ? tab_tiles : nullptr);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---- fp32 (rows, c) <-> bf16 planes (rows, planes * c_pad) --------------------------------------------------------------
__global__ void __launch_bounds__(256) k_to_planes(const float* __restrict__ x, const int* __restrict__ d_n, int cap, int c, int c_pad, int planes,
                                                   uint16_t* __restrict__ out) {
    const int n = d_n ? min(*d_n, cap) : cap;
    const long long total = (long long)n * c_pad;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i / c_pad), ch = (int)(i % c_pad);
        const float v = ch < c ? __ldg(x + (size_t)r * c + ch) : 0.f;
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        uint16_t* o = out + (size_t)r * planes * c_pad + ch;
        o[0] = *reinterpret_cast<const uint16_t*>(&h);
        if (planes == 2) {
            const __nv_bfloat16 l = __float2bfloat16_rn(v - __bfloat162float(h));
            o[c_pad] = *reinterpret_cast<const uint16_t*>(&l);
        }
    }
}
__global__ void __launch_bounds__(256) k_from_planes(const uint16_t* __restrict__ x, const int* __restrict__ d_n, int cap, int c, int planes,
                                                     float* __restrict__ out) {
    const int n = d_n ? min(*d_n, cap) : cap;
    const long long total = (long long)n * c;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i / c), ch = (int)(i % c);
        const uint16_t* p = x + (size_t)r * planes * c + ch;
        float v = __uint_as_float((uint32_t)p[0] << 16);
        if (planes == 2) v += __uint_as_float((uint32_t)p[c] << 16);
        out[i] = v;
    }
}
// HeightCompression on a planes tensor: out[b,y,x,c*D+z] = feats[i,c] (fp32 NHWC, zero on entry)
__global__ void __launch_bounds__(256) k_sparse_to_bev_planes(const uint16_t* __restrict__ feats, const int32_t* __restrict__ coords,
                                                              const int* __restrict__ d_n, int cap, int c, int planes, int D, int H, int W,
                                                              float* __restrict__ out) {
    const int n = min(*d_n, cap);
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int i = warp; i < n; i += nwarps) {
        const int4 cd = __ldg(reinterpret_cast<const int4*>(coords) + i);            // b,z,y,x
        float* dst = out + (((size_t)cd.x * H + cd.z) * W + cd.w) * ((size_t)c * D) + cd.y;
        const uint16_t* src = feats + (size_t)i * planes * c;
        for (int ch = lane; ch < c; ch += 32) {
            float v = __uint_as_float((uint32_t)__ldg(src + ch) << 16);
            if (planes == 2) v += __uint_as_float((uint32_t)__ldg(src + c + ch) << 16);
            dst[(size_t)ch * D] = v;
        }
    }
}

}  // namespace

extern "C" int dz_to_planes(const float* x, const int* d_n, int cap, int c, int c_pad, int planes, void* out, dz_stream_t stream) {
    DZ_CHECK_ARG(x && out && cap >= 1 && c >= 1 && c_pad >= c && (planes == 1 || planes == 2));
    const int blocks = max(1, min(dz_cdiv((long long)cap * c_pad, 256), DZ_NUM_SMS * 8));
    k_to_planes<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, d_n, cap, c, c_pad, planes, (uint16_t*)out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" int dz_from_planes(const void* x, const int* d_n, int cap, int c, int planes, float* out, dz_stream_t stream) {
    DZ_CHECK_ARG(x && out && cap >= 1 && c >= 1 && (planes == 1 || planes == 2));
    const int blocks = max(1, min(dz_cdiv((long long)cap * c, 256), DZ_NUM_SMS * 8));
    k_from_planes<<<blocks, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)x, d_n, cap, c, planes, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" int dz_sparse_to_bev_planes(const void* feats, const int32_t* coords, const int* d_n, int cap, int c, int planes, int B, int D,
                                       int H, int W, float* out, dz_stream_t stream) {
    DZ_CHECK_ARG(feats && coords && d_n && out && cap >= 1 && c >= 1 && (planes == 1 || planes == 2));
    (void)B;
    const int blocks = max(1, min(dz_cdiv((long long)cap * 32, 256), DZ_NUM_SMS * 8));
    k_sparse_to_bev_planes<<<blocks, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)feats, coords, d_n, cap, c, planes, D, H, W, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" int dz_spconv_fwd_planes(const void* in, int cin, int in_rows, const int32_t* tab, int K, int tab_rows, const int32_t* row_order,
                                    const int* d_n_out, int out_cap, const void* weight, const float* scale, const float* shift,
                                    const void* residual, int relu, void* out, int cout, int planes, const int32_t* tab_tiles,
                                    dz_stream_t stream) {
    DZ_CHECK_ARG(in && tab && d_n_out && weight && out && cin >= 1 && K >= 1 && K <= SB_KMAX && out_cap >= 1 && tab_rows >= out_cap);
    DZ_CHECK_ARG(planes == 1 || planes == 2);
    (void)in_rows;
    cudaStream_t st = (cudaStream_t)stream;
    const int cin_pad = cin <= 8 ? 8 : cin;
#define DZ_SB(CP, CO)                                                                                                                           \
    if (cin_pad == CP && cout == CO) {                                                                                                          \
        if (planes == 1) return launch<CP, CO, 1>(in, tab, K, tab_rows, row_order, d_n_out, out_cap, weight, scale, shift, residual, relu, out, tab_tiles, st); \
        return launch<CP, CO, 2>(in, tab, K, tab_rows, row_order, d_n_out, out_cap, weight, scale, shift, residual, relu, out, tab_tiles, st);   \
    }
    DZ_SB(8, 16) DZ_SB(16, 16) DZ_SB(16, 32) DZ_SB(32, 32) DZ_SB(32, 64) DZ_SB(64, 64) DZ_SB(64, 128) DZ_SB(128, 128)
#undef DZ_SB
    dz_set_error("dz_spconv_fwd_planes: (cin=%d, cout=%d) not instantiated", cin, cout);
    return DZ_ERR_UNSUPPORTED;
}

// spconv_tc.cu -- sparse convolution forward on the Hopper tensor cores (wgmma, TF32 operands, fp32 register accumulators).
//
// Same contract as the exact-fp32 kernel in spconv.cu (SubMConv3d / SparseConv3d + folded BatchNorm1d + bias + residual
// + ReLU, backbone3d.py:64-83,105-121) for two modes:
//   DZ_TF32   one TF32 pass.  spconv's own default keeps TF32 off (SURVEY A.4), so this mode is opt-in
//             (COMPUTE_MODE: tf32) with a stated 2e-3 tolerance.
//   DZ_TF32X3 fp32-level accuracy ("3xTF32" split): every fp32 operand is split into two TF32 pieces, x = x_hi + x_lo
//             (x_hi = RN_tf32(x), x_lo = RN_tf32(x - x_hi)), and the product is accumulated in fp32 registers as
//                 A_lo*W_hi + A_hi*W_lo + A_hi*W_hi          (the dropped A_lo*W_lo term is ~2^-22 relative)
//             which reproduces fp32 FMA results to ~1e-6 relative (tests: <= 1e-5, the bar for the fp32-exact mode,
//             SURVEY §8c).  Three MMAs per k-step instead of one: the kernel is bound by the gather, not the tensor pipe.
//
// Design: output-stationary implicit GEMM.  A CTA owns 128 output rows -- the rows order[p] of one tile of the rulebook's
// tile schedule (rows with alike neighbour masks, csrc/rulebook.cu), tiles taken heaviest-first -- and reads their
// neighbour lists from the row-major table (one 128-byte line per row).  The reduction dimension is the concatenation
// (kernel offset k, input channel c) of length K*Cin, cut into 32-float (128-byte) blocks -- for Cin = 16 one block spans
// two offsets, for Cin = 64 an offset spans two blocks -- so narrow layers still fill the MMA K dimension.  Blocks whose
// offsets no row of the tile uses are skipped (that is what the schedule maximises).  Per block, producer warps gather the
// neighbour rows into shared memory in the canonical K-major 128B-swizzled layout, one thread TMA-loads the matching
// W[cout][k-block] tile(s), and two consumer warpgroups (64 rows each) issue wgmma (M=64, N=Cout, K=8) into register
// accumulators.  The gather differs by mode:
//   tf32   two warps per stage, cp.async straight from global/L2 (zero-fill for missing neighbours); the copies arrive on
//          the stage's barrier asynchronously and the consumers fence the generic -> async proxy after their wait.
//   tf32x3 one warp per stage, through registers: LDG.128 -> hi/lo split -> two swizzled STS.128 (A_hi, A_lo tiles), then a
//          proxy fence and the arrive.  The weights are pre-split on the host and arrive as two TMA tiles.
// After the last block the accumulators go through the (then idle) pipeline buffers and warps 0-3 run the epilogue, one
// row per thread: scale/shift (+residual) -> ReLU (-> RN_tf32 for tf32) -> 128-bit stores to row order[p].  No atomics:
// deterministic, and bit-identical with or without a schedule (a row's accumulation order over k never changes).
#include "common.cuh"
#include "tc.cuh"

static constexpr int ST_ROWS = 128;
static constexpr int ST_A_BYTES = ST_ROWS * 128;        // one 32-float block for 128 rows
static constexpr int ST_KMAX = 27;

template <int COUT, bool SPLIT>
struct StCfg {
    static constexpr int PLANES = SPLIT ? 2 : 1;               // operand pieces: [A_hi | A_lo] and [W_hi | W_lo] under SPLIT
    static constexpr int W_BYTES = COUT * 128;
    static constexpr int STAGE_BYTES = PLANES * (ST_A_BYTES + W_BYTES);
    // Cout = 128: the 128 x 128 B tile is the largest stage; VoxelBackBone8x runs it only as conv_out (K = 3), VoxelResBackBone8x
    // also as spconv4 (cin = 64) and the res4 blocks (K = 27, with a residual).  Three stages still cover one step's MMAs
    static constexpr int STAGES = SPLIT ? 3 : (COUT >= 128 ? 3 : 4);
    // PW producer warps per stage: warp w gathers its 128/PW rows of the steps it = s, s+STAGES, ... into stage s = (w-8) % STAGES
    // (one warp alone cannot keep enough cp.async gathers in flight; the register gather of SPLIT keeps 8 loads per lane in
    // flight itself); warps 0-7 are the two consumer warpgroups, warps 0-3 double as the epilogue
    static constexpr int PW = SPLIT ? 1 : 2;
    static constexpr int PRODUCERS = STAGES * PW;
    static constexpr int CONSUMERS = 8;
    static constexpr int THREADS = 32 * (CONSUMERS + PRODUCERS);
    static constexpr int MIN_BLOCKS = SPLIT ? 1 : 0;                // __launch_bounds__ minimum blocks per SM (0: unspecified)
    static constexpr int ACC_LD = COUT + 4;                    // row pitch of the accumulator tile staged for the epilogue
    static constexpr int SMEM = STAGES * STAGE_BYTES + 1024 + ST_KMAX * ST_ROWS * 4 + 128 * 4 + 256;
    static_assert(ST_ROWS * ACC_LD * 4 <= STAGES * STAGE_BYTES, "accumulator staging must fit in the pipeline buffers");
};

// weight tensor maps of one launch: [W] or [W_hi, W_lo]
template <int PLANES>
struct WeightMaps { CUtensorMap m[PLANES]; };

template <int CIN_PAD, int COUT, bool SPLIT>
__global__ void __launch_bounds__(StCfg<COUT, SPLIT>::THREADS, StCfg<COUT, SPLIT>::MIN_BLOCKS)
k_spconv_tf32(const __grid_constant__ WeightMaps<StCfg<COUT, SPLIT>::PLANES> tmW, const float* __restrict__ in, int cin,
              const int32_t* __restrict__ nbr, int K, int nbr_cap, const int32_t* __restrict__ order, const int* __restrict__ d_n_out,
              int out_cap, const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ residual, int relu,
              float* __restrict__ out) {
    using Cfg = StCfg<COUT, SPLIT>;
    constexpr int PLANES = Cfg::PLANES;
    const int n = min(*d_n_out, out_cap);
    // under a tile schedule CTAs take the tiles heaviest-first (launch order ~ blockIdx order): order[nbr_cap + i]
    const int row0 = (order ? __ldg(order + nbr_cap + blockIdx.x) : (int)blockIdx.x) * ST_ROWS;
    if (row0 >= n) return;

    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    int* s_nbr = reinterpret_cast<int*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);          // [K][128]
    int* s_blocks = s_nbr + ST_KMAX * ST_ROWS;                                            // active block list (<= 108)
    uint64_t* full = reinterpret_cast<uint64_t*>(s_blocks + 124);
    uint64_t* empty = full + Cfg::STAGES;
    int* s_nb = reinterpret_cast<int*>(empty + Cfg::STAGES);
    unsigned* s_mask = reinterpret_cast<unsigned*>(s_nb + 1);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ktot = K * CIN_PAD;
    const int nb_tot = (ktot + 31) / 32;

    if (threadIdx.x == 0) {
#pragma unroll
        for (int p = 0; p < PLANES; ++p) tc::prefetch_tmap(&tmW.m[p]);
        for (int s = 0; s < Cfg::STAGES; ++s) { tc::mbar_init(full + s, 32 * Cfg::PW + 1); tc::mbar_init(empty + s, Cfg::CONSUMERS); }
        tc::fence_barrier_init();
        *s_mask = 0u;
    }
    __syncthreads();
    // ---- neighbour rows of this tile + which offsets are populated
    if (warp < 4) {
        const int r = row0 + threadIdx.x;
        // table row of this tile position (row-major table, one 128-byte line per output row; order[pos] under a schedule)
        const int src = r < n ? (order ? __ldg(order + r) : r) : -1;
        int v[ST_KMAX];
        {
            int w[28];
            const int4* rowp = reinterpret_cast<const int4*>(nbr) + (size_t)(src < 0 ? 0 : src) * 8;
#pragma unroll
            for (int q = 0; q < 7; ++q) {
                const int4 t4 = src >= 0 ? __ldg(rowp + q) : make_int4(-1, -1, -1, -1);
                w[4 * q] = t4.x; w[4 * q + 1] = t4.y; w[4 * q + 2] = t4.z; w[4 * q + 3] = t4.w;
            }
#pragma unroll
            for (int k = 0; k < ST_KMAX; ++k) v[k] = k < K ? w[k] : -1;
        }
        unsigned mine = 0;
#pragma unroll
        for (int k = 0; k < ST_KMAX; ++k) {
            if (k < K) s_nbr[k * ST_ROWS + threadIdx.x] = v[k];
            mine |= (v[k] >= 0 ? 1u : 0u) << k;
        }
        mine = __reduce_or_sync(0xffffffffu, mine);
        if (lane == 0 && mine) atomicOr(s_mask, mine);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned mask = *s_mask;
        int nb = 0;
        for (int kb = 0; kb < nb_tot; ++kb) {
            int k_lo = (kb * 32) / CIN_PAD, k_hi = min(K - 1, (kb * 32 + 31) / CIN_PAD);
            bool act = false;
            for (int k = k_lo; k <= k_hi; ++k) act |= (mask >> k) & 1u;
            if (act) s_blocks[nb++] = kb;
        }
        *s_nb = nb;
    }
    __syncthreads();
    const int nb = *s_nb;

    if (warp >= Cfg::CONSUMERS) {
        // ================= producers: warp w fills rows [part*RPW, (part+1)*RPW) of stage s for the steps s, s+STAGES, ... ===
        constexpr int RPW = ST_ROWS / Cfg::PW;      // rows per producer warp
        constexpr int RPL = RPW / 4;                // rows per 8-lane group
        const int j = lane & 7;                     // 16-byte chunk inside the 128-byte row
        const int rg = lane >> 3;                   // lane covers chunk j of rows rbase .. rbase+RPL-1
        const int s = (warp - Cfg::CONSUMERS) % Cfg::STAGES, part = (warp - Cfg::CONSUMERS) / Cfg::STAGES;
        const int rbase = part * RPW + rg * RPL;
        unsigned char* sa = smem + s * Cfg::STAGE_BYTES;
        for (int it = s, round = 0; it < nb; it += Cfg::STAGES, ++round) {
            const int kb = s_blocks[it];
            tc::mbar_wait(empty + s, (round & 1) ^ 1);
            if (part == 0 && lane == 0) {
                tc::mbar_arrive_expect_tx(full + s, PLANES * Cfg::W_BYTES);
#pragma unroll
                for (int p = 0; p < PLANES; ++p) tc::tma_load_2d(sa + PLANES * ST_A_BYTES + p * Cfg::W_BYTES, &tmW.m[p], full + s, kb * 32, 0);
            }
            const int kidx = kb * 32 + j * 4;       // position in the concatenated (offset, channel) dimension
            const int k = kidx / CIN_PAD, c = kidx % CIN_PAD;
            const bool k_ok = k < K;
            const int4* nb_k = reinterpret_cast<const int4*>(s_nbr + (k_ok ? k : 0) * ST_ROWS + rbase);
            const float* in_c = in + c;
            if constexpr (!SPLIT) {
                const uint32_t sa_u = tc::smem_u32(sa);
#pragma unroll
                for (int i0 = 0; i0 < RPL; i0 += 4) {
                    const int4 nq = nb_k[i0 / 4];
                    const int rows4[4] = {nq.x, nq.y, nq.z, nq.w};
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int src_row = k_ok ? rows4[u] : -1;
                        const int r = rbase + i0 + u;   // tile row: swizzle atom r/8, row-in-atom r%8
                        const int rr = r & 7;
                        const uint32_t dst = sa_u + (uint32_t)((r >> 3) * 1024 + rr * 128 + ((j ^ rr) << 4));
                        if (CIN_PAD >= 16) {
                            const bool ok = src_row >= 0;
                            tc::cp_async16_zfill(dst, ok ? (const void*)(in_c + (size_t)src_row * cin) : (const void*)in, ok);
                        } else {
                            // first layer (cin = 5 padded to 8): rows are not 16-byte aligned -> 4-byte copies
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                const bool ok = src_row >= 0 && (c + e) < cin;
                                tc::cp_async4_zfill(dst + 4 * e, ok ? (const void*)(in_c + (size_t)src_row * cin + e) : (const void*)in, ok);
                            }
                        }
                    }
                }
                tc::cp_async_mbar_arrive_noinc(full + s);
            } else {
                unsigned char* sa_lo = sa + ST_A_BYTES;
#pragma unroll 1
                for (int i0 = 0; i0 < RPL; i0 += 8) {
                    float4 v[8];
                    const int4 n0 = nb_k[i0 / 4], n1 = nb_k[i0 / 4 + 1];
                    const int rows8[8] = {n0.x, n0.y, n0.z, n0.w, n1.x, n1.y, n1.z, n1.w};
#pragma unroll
                    for (int u = 0; u < 8; ++u) {                       // 8 independent 128-bit loads in flight per lane
                        const int src_row = k_ok ? rows8[u] : -1;
                        v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (src_row >= 0) {
                            if (CIN_PAD >= 16) v[u] = __ldg(reinterpret_cast<const float4*>(in_c + (size_t)src_row * cin));
                            else {
                                const float* p = in_c + (size_t)src_row * cin;     // cin = 5: unaligned rows, scalar loads
                                if (c + 0 < cin) v[u].x = __ldg(p + 0);
                                if (c + 1 < cin) v[u].y = __ldg(p + 1);
                                if (c + 2 < cin) v[u].z = __ldg(p + 2);
                                if (c + 3 < cin) v[u].w = __ldg(p + 3);
                            }
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        // row r = rg*32 + i0 + u: 8-row group (r>>3) = rg*4 + i0/8, row in group = u
                        const uint32_t off = (uint32_t)((rg * 4 + (i0 >> 3)) * 1024 + u * 128 + ((j ^ u) << 4));
                        float4 hi, lo;
                        hi.x = tc::rna_tf32(v[u].x); hi.y = tc::rna_tf32(v[u].y); hi.z = tc::rna_tf32(v[u].z); hi.w = tc::rna_tf32(v[u].w);
                        lo.x = tc::rna_tf32(v[u].x - hi.x); lo.y = tc::rna_tf32(v[u].y - hi.y);      // RN (the tensor core would truncate)
                        lo.z = tc::rna_tf32(v[u].z - hi.z); lo.w = tc::rna_tf32(v[u].w - hi.w);
                        *reinterpret_cast<float4*>(sa + off) = hi;
                        *reinterpret_cast<float4*>(sa_lo + off) = lo;
                    }
                }
                tc::fence_proxy_async();                  // generic-proxy smem writes -> visible to the tensor core (async proxy)
                tc::mbar_arrive(full + s);
            }
        }
    } else {
        // ================= consumers: warpgroup g accumulates rows [64g, 64g+64) of the tile =================
        const int g = warp >> 2;
        float acc[COUT / 2];
#pragma unroll
        for (int i = 0; i < COUT / 2; ++i) acc[i] = 0.f;
        for (int it = 0; it < nb; ++it) {
            const int s = it % Cfg::STAGES;
            tc::mbar_wait(full + s, (it / Cfg::STAGES) & 1);
            if constexpr (!SPLIT) tc::fence_proxy_async();      // cp.async (generic proxy) writes -> tensor-core (async proxy) reads
            const uint32_t sa = tc::smem_u32(smem + s * Cfg::STAGE_BYTES) + g * 64 * 128;
            const uint32_t sw = tc::smem_u32(smem + s * Cfg::STAGE_BYTES) + PLANES * ST_A_BYTES;
            const uint64_t a_hi = tc::smem_desc_sw128(sa), w_hi = tc::smem_desc_sw128(sw);
            tc::wgmma_fence();
            if constexpr (!SPLIT) {
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) tc::wgmma<COUT, tc::K_TF32>(acc, a_hi + (uint64_t)(kk * 2), w_hi + (uint64_t)(kk * 2), 1u);
            } else {
                const uint64_t a_lo = tc::smem_desc_sw128(sa + ST_A_BYTES), w_lo = tc::smem_desc_sw128(sw + Cfg::W_BYTES);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    const uint64_t o = (uint64_t)(kk * 2);
                    tc::wgmma<COUT, tc::K_TF32>(acc, a_lo + o, w_hi + o, 1u);      // small terms first
                    tc::wgmma<COUT, tc::K_TF32>(acc, a_hi + o, w_lo + o, 1u);
                    tc::wgmma<COUT, tc::K_TF32>(acc, a_hi + o, w_hi + o, 1u);
                }
            }
            tc::wgmma_commit();
            tc::wgmma_wait_one();                       // this step's MMAs stay in flight; the previous step's stage is free
            __syncwarp();
            if (lane == 0 && it > 0) tc::mbar_arrive(empty + (it - 1) % Cfg::STAGES);
        }
        tc::wgmma_wait_all();
        __syncwarp();
        if (lane == 0 && nb > 0) tc::mbar_arrive(empty + (nb - 1) % Cfg::STAGES);
        // every stage has been consumed: the pipeline buffers hold the accumulator tile for the epilogue
        float* stg = reinterpret_cast<float*>(smem);
        tc::named_sync(1, 32 * Cfg::CONSUMERS);
        tc::acc_to_smem<COUT>(acc, stg, Cfg::ACC_LD, g * 64);
        tc::named_sync(1, 32 * Cfg::CONSUMERS);
        if (warp < 4) {
            // ================= epilogue: thread = tile row =================
            const int pos = row0 + threadIdx.x;     // tile position; the output row is order[pos] under a tile schedule
            const int r = pos < n ? (order ? __ldg(order + pos) : pos) : n;
#pragma unroll 1
            for (int c0 = 0; c0 < COUT; c0 += 32) {
                float v[32];
                if (c0 + 32 <= COUT) tc::smem_row32(stg, Cfg::ACC_LD, threadIdx.x, c0, v);
                else { for (int i = 0; i < 16; ++i) v[i] = stg[threadIdx.x * Cfg::ACC_LD + c0 + i]; }
                if (r < n) {
#pragma unroll
                    for (int jj = 0; jj < 32; jj += 4) {
                        const int ch = c0 + jj;
                        if (ch >= COUT) break;
                        float4 o = nb > 0 ? make_float4(v[jj], v[jj + 1], v[jj + 2], v[jj + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
                        if (scale) { float4 sc = __ldg(reinterpret_cast<const float4*>(scale + ch)); o.x *= sc.x; o.y *= sc.y; o.z *= sc.z; o.w *= sc.w; }
                        if (shift) { float4 sh = __ldg(reinterpret_cast<const float4*>(shift + ch)); o.x += sh.x; o.y += sh.y; o.z += sh.z; o.w += sh.w; }
                        if (residual) {
                            float4 rr = __ldg(reinterpret_cast<const float4*>(residual + (size_t)r * COUT + ch));
                            o.x += rr.x; o.y += rr.y; o.z += rr.z; o.w += rr.w;
                        }
                        if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
                        if constexpr (!SPLIT) {
                            // round-to-nearest to TF32: the next layer's truncating tensor-core read is then exact (no toward-zero bias)
                            o.x = tc::rna_tf32(o.x); o.y = tc::rna_tf32(o.y); o.z = tc::rna_tf32(o.z); o.w = tc::rna_tf32(o.w);
                        }
                        *reinterpret_cast<float4*>(out + (size_t)r * COUT + ch) = o;
                    }
                }
            }
        }
    }
}

// weight layout: tf32 (cout, K*cin_pad) row-major, cin_pad = 8 for cin <= 8 else cin; tf32x3 (2, cout, K*cin_pad):
// [0] = RN_tf32(W), [1] = RN_tf32(W - W_hi).
// (A TMA tile::gather4 producer was built and measured 1.6x slower than the cp.async gather for 128-byte rows -- the TMA unit
// has a per-row cost -- and a hybrid LSU+TMA split gave no gain.  Both were removed.)
template <int CIN_PAD, int COUT, bool SPLIT>
static int launch(const float* in, int cin, const int32_t* nbr, int K, int nbr_cap, const int32_t* order, const int* d_n_out, int out_cap,
                  const float* weight, const float* scale, const float* shift, const float* residual, int relu, float* out, cudaStream_t st) {
    using Cfg = StCfg<COUT, SPLIT>;
    tc::EncodeTiledFn enc = tc::get_encode_tiled();
    if (!enc) { dz_set_error("cuTensorMapEncodeTiled unavailable"); return DZ_ERR_CUDA; }
    WeightMaps<Cfg::PLANES> tm;
    const cuuint64_t ktot = (cuuint64_t)K * CIN_PAD;
    for (int p = 0; p < Cfg::PLANES; ++p) {
        cuuint64_t dims[2] = {ktot, (cuuint64_t)COUT};
        cuuint64_t strides[1] = {ktot * 4};
        cuuint32_t box[2] = {32, (cuuint32_t)COUT};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&tm.m[p], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)(weight + (size_t)p * COUT * ktot), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(W) failed: %d", (int)r); return DZ_ERR_CUDA; }
    }
    static bool configured = false;
    if (!configured) {
        DZ_CUDA(cudaFuncSetAttribute(k_spconv_tf32<CIN_PAD, COUT, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
        configured = true;
    }
    k_spconv_tf32<CIN_PAD, COUT, SPLIT><<<dz_cdiv(out_cap, ST_ROWS), Cfg::THREADS, Cfg::SMEM, st>>>(tm, in, cin, nbr, K, nbr_cap, order, d_n_out,
                                                                                                  out_cap, scale, shift, residual, relu, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

int dz_spconv_fwd_tc(const float* in, int cin, int in_rows, const int32_t* nbr, int K, int nbr_cap, const int32_t* order, const int* d_n_out, int out_cap,
                     const float* weight, const float* scale, const float* shift, const float* residual, int relu, float* out,
                     int cout, int mode, cudaStream_t st) {
    (void)in_rows;
    if (mode != DZ_TF32 && mode != DZ_TF32X3) { dz_set_error("dz_spconv_fwd: tensor-core mode %d not built (tf32, tf32x3)", mode); return DZ_ERR_UNSUPPORTED; }
    const bool split = mode == DZ_TF32X3;
    const char* name = split ? "tf32x3" : "tf32";
    if (K > ST_KMAX) { dz_set_error("dz_spconv_fwd(%s): K=%d > 27", name, K); return DZ_ERR_UNSUPPORTED; }
    const int cin_pad = cin <= 8 ? 8 : cin;
#define DZ_ST(CP, CO)                                                                                                                       \
    if (cin_pad == CP && cout == CO) {                                                                                                      \
        if (split) return launch<CP, CO, true>(in, cin, nbr, K, nbr_cap, order, d_n_out, out_cap, weight, scale, shift, residual, relu, out, st); \
        return launch<CP, CO, false>(in, cin, nbr, K, nbr_cap, order, d_n_out, out_cap, weight, scale, shift, residual, relu, out, st);     \
    }
    DZ_ST(8, 16) DZ_ST(16, 16) DZ_ST(16, 32) DZ_ST(32, 32) DZ_ST(32, 64) DZ_ST(64, 64) DZ_ST(64, 128) DZ_ST(128, 128)
#undef DZ_ST
    dz_set_error("dz_spconv_fwd(%s): (cin=%d, cout=%d) not instantiated", name, cin, cout);
    return DZ_ERR_UNSUPPORTED;
}

// RN_tf32 (ties to even) of the first min(*d_n, cap) rows: the same bits as ops.round_tf32, non-finite values kept
__global__ void __launch_bounds__(256) k_round_tf32(const float* __restrict__ x, const int* __restrict__ d_n, int cap, int c, float* __restrict__ out) {
    const int n = d_n ? min(*d_n, cap) : cap;
    const long long total = (long long)n * c;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const uint32_t u = __float_as_uint(x[i]);
        out[i] = (u & 0x7f800000u) == 0x7f800000u ? __uint_as_float(u) : __uint_as_float((u + 0xfffu + ((u >> 13) & 1u)) & ~0x1fffu);
    }
}

extern "C" int dz_round_tf32(const float* x, const int* d_n, int cap, int c, float* out, dz_stream_t stream) {
    DZ_CHECK_ARG(x && out && cap >= 1 && c >= 1);
    const int blocks = max(1, min(dz_cdiv((long long)cap * c, 256), DZ_NUM_SMS * 8));
    k_round_tf32<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, d_n, cap, c, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// spconv_tc3.cu -- sparse convolution forward with fp32-LEVEL accuracy on the tensor cores ("3xTF32" split), sm_90a.
//
// spconv keeps TF32 off by default, so the reference arithmetic of SubMConv3d / SparseConv3d is fp32 FMA (SURVEY A.4).
// A single TF32 pass (spconv_tc.cu) has a 2^-11 input rounding; here every fp32 operand is split into two TF32 pieces,
// x = x_hi + x_lo (x_hi = RN_tf32(x), x_lo = x - x_hi exactly), and the product is accumulated in fp32 registers as
//     A_hi*W_hi + A_lo*W_hi + A_hi*W_lo            (the dropped A_lo*W_lo term is ~2^-22 relative)
// which reproduces fp32 FMA results to ~1e-6 relative (tests: <= 1e-5, the bar for the fp32-exact mode, SURVEY §8c) while
// the math runs on wgmma.  Three MMAs per k-step instead of one: the kernel is bound by the gather rather than by the
// tensor pipe.
//
// Structure = spconv_tc.cu (128-row tile, (offset,channel) reduction in 128-byte blocks, one producer warp per stage,
// two consumer warpgroups, epilogue from the staged accumulators) except that the gather goes through registers: LDG.128 -> split -> two
// swizzled STS.128 (A_hi tile, A_lo tile); the weights are pre-split on the host and arrive by TMA.
#include "common.cuh"
#include "tc.cuh"

static constexpr int S3_ROWS = 128;
static constexpr int S3_A_BYTES = S3_ROWS * 128;
static constexpr int S3_KMAX = 27;

template <int COUT>
struct S3Cfg {
    static constexpr int W_BYTES = COUT * 128;
    static constexpr int STAGE_BYTES = 2 * S3_A_BYTES + 2 * W_BYTES;
    static constexpr int STAGES = 3;
    static constexpr int CONSUMERS = 8;                          // two consumer warpgroups (64 rows each); warps 0-3 run the epilogue
    static constexpr int THREADS = 32 * (CONSUMERS + STAGES);    // warp CONSUMERS + s fills stage s
    static constexpr int ACC_LD = COUT + 4;
    static constexpr int SMEM = STAGES * STAGE_BYTES + 1024 + S3_KMAX * S3_ROWS * 4 + 128 * 4 + 256;
    static_assert(S3_ROWS * ACC_LD * 4 <= STAGES * STAGE_BYTES, "accumulator staging must fit in the pipeline buffers");
};

template <int CIN_PAD, int COUT>
__global__ void __launch_bounds__(S3Cfg<COUT>::THREADS, 1)
k_spconv_3xtf32(const __grid_constant__ CUtensorMap tmWhi, const __grid_constant__ CUtensorMap tmWlo, const float* __restrict__ in, int cin,
                const int32_t* __restrict__ nbr, int K, int nbr_cap, const int32_t* __restrict__ order, const int* __restrict__ d_n_out, int out_cap,
                const float* __restrict__ scale, const float* __restrict__ shift, const float* __restrict__ residual, int relu,
                float* __restrict__ out) {
    using Cfg = S3Cfg<COUT>;
    const int n = min(*d_n_out, out_cap);
    // under a tile schedule CTAs take the tiles heaviest-first (launch order ~ blockIdx order): order[nbr_cap + i]
    const int row0 = (order ? __ldg(order + nbr_cap + blockIdx.x) : (int)blockIdx.x) * S3_ROWS;
    if (row0 >= n) return;

    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    int* s_nbr = reinterpret_cast<int*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
    int* s_blocks = s_nbr + S3_KMAX * S3_ROWS;
    uint64_t* full = reinterpret_cast<uint64_t*>(s_blocks + 124);
    uint64_t* empty = full + Cfg::STAGES;
    int* s_nb = reinterpret_cast<int*>(empty + Cfg::STAGES);
    unsigned* s_mask = reinterpret_cast<unsigned*>(s_nb + 1);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nb_tot = (K * CIN_PAD + 31) / 32;

    if (threadIdx.x == 0) {
        tc::prefetch_tmap(&tmWhi);
        tc::prefetch_tmap(&tmWlo);
        for (int s = 0; s < Cfg::STAGES; ++s) { tc::mbar_init(full + s, 32 + 1); tc::mbar_init(empty + s, Cfg::CONSUMERS); }
        tc::fence_barrier_init();
        *s_mask = 0u;
    }
    __syncthreads();
    if (warp < 4) {
        const int r = row0 + threadIdx.x;
        // table row of this tile position (row-major table, one 128-byte line per output row; order[pos] under a schedule)
        const int src = r < n ? (order ? __ldg(order + r) : r) : -1;
        int v[S3_KMAX];
        {
            int w[28];
            const int4* rowp = reinterpret_cast<const int4*>(nbr) + (size_t)(src < 0 ? 0 : src) * 8;
#pragma unroll
            for (int q = 0; q < 7; ++q) {
                const int4 t4 = src >= 0 ? __ldg(rowp + q) : make_int4(-1, -1, -1, -1);
                w[4 * q] = t4.x; w[4 * q + 1] = t4.y; w[4 * q + 2] = t4.z; w[4 * q + 3] = t4.w;
            }
#pragma unroll
            for (int k = 0; k < S3_KMAX; ++k) v[k] = k < K ? w[k] : -1;
        }
        unsigned mine = 0;
#pragma unroll
        for (int k = 0; k < S3_KMAX; ++k) {
            if (k < K) s_nbr[k * S3_ROWS + threadIdx.x] = v[k];
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
        // ================= producers: warp w fills stage w (A_hi, A_lo through registers; W_hi, W_lo by TMA) ==========
        const int j = lane & 7, rg = lane >> 3;         // lane covers chunk j of rows rg*32 .. rg*32+31
        const int s = warp - Cfg::CONSUMERS;
        unsigned char* sa = smem + s * Cfg::STAGE_BYTES;
        unsigned char* sa_lo = sa + S3_A_BYTES;
        for (int it = s, round = 0; it < nb; it += Cfg::STAGES, ++round) {
            const int kb = s_blocks[it];
            tc::mbar_wait(empty + s, (round & 1) ^ 1);
            if (lane == 0) {
                tc::mbar_arrive_expect_tx(full + s, 2 * Cfg::W_BYTES);
                tc::tma_load_2d(sa + 2 * S3_A_BYTES, &tmWhi, full + s, kb * 32, 0);
                tc::tma_load_2d(sa + 2 * S3_A_BYTES + Cfg::W_BYTES, &tmWlo, full + s, kb * 32, 0);
            }
            const int kidx = kb * 32 + j * 4;
            const int k = kidx / CIN_PAD, c = kidx % CIN_PAD;
            const bool k_ok = k < K;
            const int4* nb_k = reinterpret_cast<const int4*>(s_nbr + (k_ok ? k : 0) * S3_ROWS + rg * 32);
            const float* in_c = in + c;
#pragma unroll 1
            for (int i0 = 0; i0 < 32; i0 += 8) {
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
    } else {
        // ================= consumers: warpgroup g accumulates rows [64g, 64g+64) of the tile =================
        const int g = warp >> 2;
        float acc[COUT / 2];
#pragma unroll
        for (int i = 0; i < COUT / 2; ++i) acc[i] = 0.f;
        for (int it = 0; it < nb; ++it) {
            const int s = it % Cfg::STAGES;
            tc::mbar_wait(full + s, (it / Cfg::STAGES) & 1);
            const uint32_t sa = tc::smem_u32(smem + s * Cfg::STAGE_BYTES) + g * 64 * 128;
            const uint32_t sw = tc::smem_u32(smem + s * Cfg::STAGE_BYTES) + 2 * S3_A_BYTES;
            const uint64_t a_hi = tc::smem_desc_sw128(sa), a_lo = tc::smem_desc_sw128(sa + S3_A_BYTES);
            const uint64_t w_hi = tc::smem_desc_sw128(sw), w_lo = tc::smem_desc_sw128(sw + Cfg::W_BYTES);
            tc::wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint64_t o = (uint64_t)(kk * 2);
                tc::wgmma<COUT, tc::K_TF32>(acc, a_lo + o, w_hi + o, 1u);      // small terms first
                tc::wgmma<COUT, tc::K_TF32>(acc, a_hi + o, w_lo + o, 1u);
                tc::wgmma<COUT, tc::K_TF32>(acc, a_hi + o, w_hi + o, 1u);
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
                        *reinterpret_cast<float4*>(out + (size_t)r * COUT + ch) = o;
                    }
                }
            }
        }
    }
}

template <int CIN_PAD, int COUT>
static int launch3(const CUtensorMap& hi, const CUtensorMap& lo, const float* in, int cin, const int32_t* nbr, int K, int nbr_cap,
                   const int32_t* order, const int* d_n_out, int out_cap, const float* scale, const float* shift, const float* residual, int relu, float* out,
                   cudaStream_t st) {
    using Cfg = S3Cfg<COUT>;
    static bool configured = false;
    if (!configured) {
        DZ_CUDA(cudaFuncSetAttribute(k_spconv_3xtf32<CIN_PAD, COUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
        configured = true;
    }
    k_spconv_3xtf32<CIN_PAD, COUT><<<dz_cdiv(out_cap, S3_ROWS), Cfg::THREADS, Cfg::SMEM, st>>>(hi, lo, in, cin, nbr, K, nbr_cap, order, d_n_out, out_cap,
                                                                                             scale, shift, residual, relu, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// weight layout: (2, cout, K*cin_pad): [0] = RN_tf32(W), [1] = RN_tf32(W - W_hi)
int dz_spconv_fwd_tc3(const float* in, int cin, const int32_t* nbr, int K, int nbr_cap, const int32_t* order, const int* d_n_out, int out_cap,
                      const float* weight, const float* scale, const float* shift, const float* residual, int relu, float* out,
                      int cout, cudaStream_t st) {
    if (K > S3_KMAX) { dz_set_error("dz_spconv_fwd(tf32x3): K=%d > 27", K); return DZ_ERR_UNSUPPORTED; }
    const int cin_pad = cin <= 8 ? 8 : cin;
    tc::EncodeTiledFn enc = tc::get_encode_tiled();
    if (!enc) { dz_set_error("cuTensorMapEncodeTiled unavailable"); return DZ_ERR_CUDA; }
    CUtensorMap tm[2];
    cuuint64_t ktot = (cuuint64_t)K * cin_pad;
    for (int h = 0; h < 2; ++h) {
        cuuint64_t dims[2] = {ktot, (cuuint64_t)cout};
        cuuint64_t strides[1] = {ktot * 4};
        cuuint32_t box[2] = {32, (cuuint32_t)cout};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&tm[h], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)(weight + (size_t)h * cout * ktot), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(W) failed: %d", (int)r); return DZ_ERR_CUDA; }
    }
#define DZ_S3(CP, CO) return launch3<CP, CO>(tm[0], tm[1], in, cin, nbr, K, nbr_cap, order, d_n_out, out_cap, scale, shift, residual, relu, out, st)
    if (cin_pad == 8 && cout == 16) DZ_S3(8, 16);
    if (cin_pad == 16 && cout == 16) DZ_S3(16, 16);
    if (cin_pad == 16 && cout == 32) DZ_S3(16, 32);
    if (cin_pad == 32 && cout == 32) DZ_S3(32, 32);
    if (cin_pad == 32 && cout == 64) DZ_S3(32, 64);
    if (cin_pad == 64 && cout == 64) DZ_S3(64, 64);
    if (cin_pad == 64 && cout == 128) DZ_S3(64, 128);
    if (cin_pad == 128 && cout == 128) DZ_S3(128, 128);
#undef DZ_S3
    dz_set_error("dz_spconv_fwd(tf32x3): (cin=%d, cout=%d) not instantiated", cin, cout);
    return DZ_ERR_UNSUPPORTED;
}

// attention_tc.cu -- multi-head attention core on the Hopper tensor cores (wgmma, TF32 operands, fp32 register accumulators).
//
// Replaces bmm(q,k^T) + key_padding masked_fill(-inf) + softmax + bmm(.,v) of multi_head_attention_forward
// (refining/detzero_refine/models/modules/transformer/multi_head_attention.py:266-286), head_dim 32, without ever
// materialising the (B*H, Pq, Pk) score tensor.
//
// One CTA = one (batch, head) x one tile of 128 queries, ONE pass over the keys in blocks of 128 (online softmax):
//   warps 0-7  : two consumer warpgroups, 64 queries each.  Per key block: S = Q K^T (wgmma M64 N128 K8 x 4, registers), masked
//                row maxima / exp2 in registers (a row's 128 scores live in the 4 threads of a lane quad), P to shared memory
//                in the K-major SW128 A-operand layout, O = O * exp2(m_old - m_new) + P V (wgmma M64 N32 K8 x 16, registers).
//   warps 8-11 : loaders.  Warp 8 lane 0 TMA-loads the Q tile once and the K blocks (rows of 128 B = one head slice,
//                SWIZZLE_128B = K-major B operand); each warp transposes one 32-key k-block of V into V^T through registers
//                (TF32 wgmma takes K-major operands only, and for P V the keys are the reduction dimension).
#include <stdlib.h>
#include "common.cuh"
#include "tc.cuh"

static constexpr int AT_M = 128;            // queries per CTA
static constexpr int AT_N = 128;            // keys per block
static constexpr int AT_D = 32;             // head dim
static constexpr int AT_TILE = AT_M * 128;  // 16 KB: 128 rows x 128 B
static constexpr int AT_CONSUMERS = 8;
static constexpr int AT_THREADS = 32 * (AT_CONSUMERS + 4);

// 2^x on the MUFU pipe, one instruction (its arguments here are <= 0 and results land in (0, 1], where ex2.approx is good
// to 2 ulp -- far inside the TF32 tolerance of this mode)
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

struct AtSmem {
    static constexpr int Q = 0;
    static constexpr int K = AT_TILE;                    // 2 stages
    static constexpr int VT = K + 2 * AT_TILE;           // 2 stages of 4 k-blocks x (32 rows x 128 B) = 16 KB each
    static constexpr int P = VT + 2 * AT_TILE;           // per warpgroup: 4 k-blocks x (64 rows x 128 B) = 32 KB
    static constexpr int MASK = P + 4 * AT_TILE;         // per warpgroup: 4 words = the 128 keys of the block (1 = masked)
    static constexpr int BARS = MASK + 64;
    static constexpr int TOTAL = BARS + 256 + 1024;
};

__global__ void __launch_bounds__(AT_THREADS, 1)
k_attention_tf32(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const float* __restrict__ v, int ldv,
                 const unsigned char* __restrict__ kpm, int Pq, int Pk, int H, float* __restrict__ out, int ldo) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + AtSmem::BARS);
    uint64_t* q_full = bars + 0;
    uint64_t* k_full = bars + 1;      // [2]
    uint64_t* k_empty = bars + 3;     // [2]
    uint64_t* v_full = bars + 5;      // [2]
    uint64_t* v_empty = bars + 7;     // [2]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bh = blockIdx.y, b = bh / H, h = bh % H;
    const int q0 = blockIdx.x * AT_M;
    const int nblk = (Pk + AT_N - 1) / AT_N;

    if (threadIdx.x == 0) {
        tc::prefetch_tmap(&tmQ);
        tc::prefetch_tmap(&tmK);
        tc::mbar_init(q_full, 1);
        for (int i = 0; i < 2; ++i) {
            tc::mbar_init(k_full + i, 1); tc::mbar_init(k_empty + i, AT_CONSUMERS);
            tc::mbar_init(v_full + i, 4); tc::mbar_init(v_empty + i, AT_CONSUMERS);
        }
        tc::fence_barrier_init();
    }
    __syncthreads();

    if (warp >= AT_CONSUMERS) {
        // ============================== loaders ==============================
        const int kk = warp - AT_CONSUMERS;                         // this warp's k-block (32 keys) of every V block
        if (kk == 0 && lane == 0) {
            tc::mbar_arrive_expect_tx(q_full, AT_TILE);
            tc::tma_load_2d(smem + AtSmem::Q, &tmQ, q_full, h * AT_D, b * Pq + q0);
        }
        for (int j = 0; j < nblk; ++j) {
            const int st = j & 1;
            if (kk == 0 && lane == 0) {
                tc::mbar_wait(k_empty + st, ((j >> 1) & 1) ^ 1);
                tc::mbar_arrive_expect_tx(k_full + st, AT_TILE);
                tc::tma_load_2d(smem + AtSmem::K + st * AT_TILE, &tmK, k_full + st, h * AT_D, b * Pk + j * AT_N);
            }
            tc::mbar_wait(v_empty + st, ((j >> 1) & 1) ^ 1);
            unsigned char* vt = smem + AtSmem::VT + st * AT_TILE;
            // lane handles key kk*32 + lane ; 8 float4 per key ; writes V^T[d][key] swizzled
            const int key = kk * 32 + lane, kg = j * AT_N + key;
            const float* vp = v + ((size_t)b * Pk + kg) * ldv + h * AT_D;
            float4 x[8];
#pragma unroll
            for (int d4 = 0; d4 < 8; ++d4) x[d4] = (kg < Pk) ? __ldg(reinterpret_cast<const float4*>(vp) + d4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int d4 = 0; d4 < 8; ++d4) {
                const float e[4] = {x[d4].x, x[d4].y, x[d4].z, x[d4].w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int d = d4 * 4 + i;                       // row of V^T
                    // k-block kk (32 keys = 128 B), row d: (d>>3)*1024 + (d&7)*128, 16-byte chunk (lane>>2) ^ (d&7)
                    const uint32_t off = (uint32_t)(kk * 4096 + (d >> 3) * 1024 + (d & 7) * 128 + (((lane >> 2) ^ (d & 7)) << 4) + (lane & 3) * 4);
                    *reinterpret_cast<float*>(vt + off) = e[i];
                }
            }
            tc::fence_proxy_async();
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(v_full + st);
        }
    } else {
        // ============================== consumers: warpgroup g = queries [64g, 64g+64) ==============================
        const int g = warp >> 2, w = warp & 3, tid = threadIdx.x & 127;
        const int rl = 16 * w + (lane >> 2);                        // this thread's rows: rl and rl + 8 of the warpgroup
        const unsigned char* mrow = kpm ? kpm + (size_t)b * Pk : nullptr;
        uint32_t* mwords = reinterpret_cast<uint32_t*>(smem + AtSmem::MASK) + g * 4;
        unsigned char* pg = smem + AtSmem::P + g * 2 * AT_TILE;
        const uint64_t qdesc = tc::smem_desc_sw128(tc::smem_u32(smem + AtSmem::Q) + g * 64 * 128);
        const float LOG2E = 1.4426950408889634f;
        float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
        float o[AT_D / 2];
#pragma unroll
        for (int i = 0; i < AT_D / 2; ++i) o[i] = 0.f;
        tc::mbar_wait(q_full, 0);
        for (int j = 0; j < nblk; ++j) {
            const int st = j & 1;
            // key mask of the block: one key per thread, one ballot word per warp
            {
                const int key = j * AT_N + tid;
                const bool mk = key >= Pk || (mrow && mrow[key]);
                const uint32_t word = __ballot_sync(0xffffffffu, mk);
                if (lane == 0) mwords[w] = word;
            }
            // S = Q K_j^T
            float s[AT_N / 2];
            tc::mbar_wait(k_full + st, (j >> 1) & 1);
            const uint64_t kdesc = tc::smem_desc_sw128(tc::smem_u32(smem + AtSmem::K + st * AT_TILE));
            tc::wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) tc::wgmma<AT_N, tc::K_TF32>(s, qdesc + (uint64_t)(kk * 2), kdesc + (uint64_t)(kk * 2), kk ? 1u : 0u);
            tc::wgmma_commit();
            tc::wgmma_wait_all();
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(k_empty + st);
            tc::named_sync(2 + g, 128);                             // mask words of this block are visible
            uint32_t mw[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) mw[i] = mwords[i];
            // masked row maxima (column of s[4c + 2r + e] = 8c + 2(lane%4) + e)
            float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int c = 0; c < AT_N / 8; ++c)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = 8 * c + 2 * (lane & 3) + e;
                    if ((mw[col >> 5] >> (col & 31)) & 1u) { s[4 * c + e] = -INFINITY; s[4 * c + 2 + e] = -INFINITY; }
                    mx[0] = fmaxf(mx[0], s[4 * c + e]);
                    mx[1] = fmaxf(mx[1], s[4 * c + 2 + e]);
                }
            float alpha[2], ms[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
                const float m_new = fmaxf(m_run[r], mx[r]);
                alpha[r] = (m_run[r] == -INFINITY) ? 0.f : ex2_approx((m_run[r] - m_new) * LOG2E);
                ms[r] = m_new == -INFINITY ? 0.f : m_new * LOG2E;   // a row with every key so far masked keeps P = 0
                m_run[r] = m_new;
            }
            // P = exp2(S - m) -> shared memory (k-block c/4, row rl + 8r, SW128)
            float psum[2] = {0.f, 0.f};
#pragma unroll
            for (int c = 0; c < AT_N / 8; ++c)
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const float p0 = ex2_approx(fmaf(s[4 * c + 2 * r], LOG2E, -ms[r]));
                    const float p1 = ex2_approx(fmaf(s[4 * c + 2 * r + 1], LOG2E, -ms[r]));
                    psum[r] += p0 + p1;
                    const int row = rl + 8 * r, cc = (8 * c + 2 * (lane & 3)) & 31;
                    const uint32_t off = (uint32_t)((c >> 2) * 8192 + (row >> 3) * 1024 + (row & 7) * 128 + (((cc >> 2) ^ (row & 7)) << 4) + (cc & 3) * 4);
                    *reinterpret_cast<float2*>(pg + off) = make_float2(p0, p1);
                }
#pragma unroll
            for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * alpha[r] + psum[r];
#pragma unroll
            for (int c = 0; c < AT_D / 8; ++c)
#pragma unroll
                for (int r = 0; r < 2; ++r) { o[4 * c + 2 * r] *= alpha[r]; o[4 * c + 2 * r + 1] *= alpha[r]; }
            tc::fence_proxy_async();                                // P (generic-proxy writes) -> wgmma operand reads
            tc::named_sync(2 + g, 128);
            // O += P V_j
            tc::mbar_wait(v_full + st, (j >> 1) & 1);
            const uint32_t pa = tc::smem_u32(pg), va = tc::smem_u32(smem + AtSmem::VT + st * AT_TILE);
            tc::wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 16; ++kk) {
                const uint64_t pdesc = tc::smem_desc_sw128(pa + (kk >> 2) * 8192) + (uint64_t)((kk & 3) * 2);
                const uint64_t vdesc = tc::smem_desc_sw128(va + (kk >> 2) * 4096) + (uint64_t)((kk & 3) * 2);
                tc::wgmma<AT_D, tc::K_TF32>(o, pdesc, vdesc, 1u);
            }
            tc::wgmma_commit();
            tc::wgmma_wait_all();
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(v_empty + st);
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
            l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
            const int qi = q0 + g * 64 + rl + 8 * r;
            if (qi < Pq) {
                float* op = out + ((size_t)b * Pq + qi) * ldo + h * AT_D;
                const float inv = 1.f / l_run[r];                   // l == 0 (every key masked): NaN, like softmax of all -inf
#pragma unroll
                for (int c = 0; c < AT_D / 8; ++c) {
                    float2 x = make_float2(o[4 * c + 2 * r] * inv, o[4 * c + 2 * r + 1] * inv);
                    if (l_run[r] == 0.f) x = make_float2(NAN, NAN);
                    *reinterpret_cast<float2*>(op + 8 * c + 2 * (lane & 3)) = x;
                }
            }
        }
    }
}

int dz_attention_fwd_tc(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const unsigned char* kpm, int B,
                        int Pq, int Pk, int H, int dh, float* out, int ldo, int mode, cudaStream_t st) {
    if (mode != DZ_TF32) { dz_set_error("dz_attention_fwd: tensor-core mode %d not built (tf32 only)", mode); return DZ_ERR_UNSUPPORTED; }
    if (dh != AT_D) { dz_set_error("dz_attention_fwd(tf32): head_dim %d unsupported (32)", dh); return DZ_ERR_UNSUPPORTED; }
    if ((ldq & 3) || (ldk & 3) || (ldv & 3) || (ldo & 3) || (((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) & 15)) {
        dz_set_error("dz_attention_fwd(tf32): rows must be 16-byte aligned"); return DZ_ERR_ARG;
    }
    tc::EncodeTiledFn enc = tc::get_encode_tiled();
    if (!enc) { dz_set_error("cuTensorMapEncodeTiled unavailable"); return DZ_ERR_CUDA; }
    CUtensorMap tmQ, tmK;
    const float* ptrs[2] = {q, k};
    const int lds[2] = {ldq, ldk};
    const long long rows[2] = {(long long)B * Pq, (long long)B * Pk};
    CUtensorMap* maps[2] = {&tmQ, &tmK};
    for (int i = 0; i < 2; ++i) {
        // the head slice starts at column h*32 of a row of ld floats; the map covers the H*32 columns reachable from the base pointer
        cuuint64_t dims[2] = {(cuuint64_t)(H * AT_D), (cuuint64_t)rows[i]};
        cuuint64_t strides[1] = {(cuuint64_t)lds[i] * 4};
        cuuint32_t box[2] = {AT_D, AT_M};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(maps[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)ptrs[i], dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { dz_set_error("cuTensorMapEncodeTiled(attention %d) failed: %d", i, (int)r); return DZ_ERR_CUDA; }
    }
    static bool configured = false;
    if (!configured) {
        DZ_CUDA(cudaFuncSetAttribute(k_attention_tf32, cudaFuncAttributeMaxDynamicSharedMemorySize, AtSmem::TOTAL));
        configured = true;
    }
    dim3 grid(dz_cdiv(Pq, AT_M), B * H);
    k_attention_tf32<<<grid, AT_THREADS, AtSmem::TOTAL, st>>>(tmQ, tmK, v, ldv, kpm, Pq, Pk, H, out, ldo);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// spconv_bwd.cu -- backward of the sparse convolution on the same neighbour tables (SURVEY.md §8f row 1), exact fp32, sm_90a.
//
// The reference trains through spconv's autograd (detection/tools/train_utils.py:59-68: loss.backward() over SubMConv3d /
// SparseConv3d, backbone3d.py:64-121).  With out[o] = sum_k W[k] in[nbr[k][o]]:
//   dgrad   d_in[j]  = sum_k W[k]^T d_out[o]  over the pairs (k, j = nbr[k][o], o)  -- for a fixed k the map o -> j is injective, so
//           this is the FORWARD kernel again on the transposed table nbrT[k][j] = o with W[k]^T (dz_rulebook_transpose builds nbrT);
//           the same transposed table + its own weights is SparseInverseConv3d (backbone3d.py:72-73)
//   wgrad   dW[k]    = sum_o in[nbr[k][o]]^T (x) d_out[o]                            -- dz_spconv_wgrad (gathered A^T B per offset)
#include "common.cuh"

__global__ void __launch_bounds__(256) k_fill_i32(int32_t* __restrict__ p, size_t n, int32_t v) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}

__global__ void __launch_bounds__(256) k_nbr_transpose(const int32_t* __restrict__ nbr, int K, int cap_out, const int* __restrict__ d_n_out,
                                                       int32_t* __restrict__ nbrT, int cap_in) {
    const int n = min(*d_n_out, cap_out);
    const int k = blockIdx.y;
    for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < n; o += gridDim.x * blockDim.x) {
        const int j = __ldg(nbr + (size_t)k * cap_out + o);
        if (j >= 0 && j < cap_in) nbrT[(size_t)k * cap_in + j] = o;
    }
}

extern "C" int dz_rulebook_transpose(const int32_t* nbr, int K, int cap_out, const int* d_n_out, int32_t* nbrT, int cap_in,
                                     dz_stream_t stream) {
    DZ_CHECK_ARG(nbr && d_n_out && nbrT && K >= 1 && cap_out >= 1 && cap_in >= 1);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t tot = (size_t)K * cap_in;
    k_fill_i32<<<max(1, min(dz_cdiv((long long)tot, 256), DZ_NUM_SMS * 8)), 256, 0, st>>>(nbrT, tot, -1);
    dim3 grid(max(1, min(dz_cdiv(cap_out, 256), DZ_NUM_SMS * 4)), K);
    k_nbr_transpose<<<grid, 256, 0, st>>>(nbr, K, cap_out, d_n_out, nbrT, cap_in);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// dW[k][ci][co] += sum over the block's rows o (with j = nbr[k][o] >= 0) of in[j][ci] * dout[o][co].
// grid (row chunks, K); 256 threads; thread t owns the outputs e = t, t+256, ... of the cin x cout tile.
static constexpr int WG_ROWS = 1024;     // output rows per block
static constexpr int WG_BATCH = 16;      // pairs staged per step
__global__ void __launch_bounds__(256) k_spconv_wgrad(const float* __restrict__ in, int cin, const int32_t* __restrict__ nbr, int nbr_cap,
                                                      const int* __restrict__ d_n_out, int out_cap, const float* __restrict__ dout, int cout,
                                                      float* __restrict__ dW) {
    extern __shared__ float smem[];
    float* sa = smem;                         // [WG_BATCH][cin]
    float* sb = smem + WG_BATCH * cin;        // [WG_BATCH][cout]
    __shared__ int s_j[WG_BATCH], s_o[WG_BATCH], s_m;
    const int n = min(*d_n_out, out_cap);
    const int k = blockIdx.y;
    const int r0 = blockIdx.x * WG_ROWS, r1 = min(n, r0 + WG_ROWS);
    if (r0 >= n) return;
    const int tile = cin * cout;
    constexpr int MAXE = 64;                  // cin * cout / 256 <= 128 * 128 / 256
    float acc[MAXE];
#pragma unroll
    for (int e = 0; e < MAXE; ++e) acc[e] = 0.f;
    for (int base = r0; base < r1; base += WG_BATCH) {
        if (threadIdx.x < 32) {               // compact the valid pairs of this batch (warp 0)
            const int o = base + (int)threadIdx.x;
            const int j = (threadIdx.x < WG_BATCH && o < r1) ? __ldg(nbr + (size_t)k * nbr_cap + o) : -1;
            const unsigned bal = __ballot_sync(0xffffffffu, j >= 0);
            if (j >= 0) { const int p = __popc(bal & ((1u << threadIdx.x) - 1u)); s_j[p] = j; s_o[p] = o; }
            if (threadIdx.x == 0) s_m = __popc(bal);
        }
        __syncthreads();
        const int m = s_m;
        if (m) {
            for (int t = threadIdx.x; t < m * cin; t += 256) sa[t] = __ldg(in + (size_t)s_j[t / cin] * cin + t % cin);
            for (int t = threadIdx.x; t < m * cout; t += 256) sb[t] = __ldg(dout + (size_t)s_o[t / cout] * cout + t % cout);
            __syncthreads();
#pragma unroll
            for (int e = 0; e < MAXE; ++e) {
                const int idx = threadIdx.x + e * 256;
                if (idx < tile) {
                    const int ci = idx / cout, co = idx % cout;
                    float a = acc[e];
                    for (int p = 0; p < m; ++p) a = fmaf(sa[p * cin + ci], sb[p * cout + co], a);
                    acc[e] = a;
                }
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int e = 0; e < MAXE; ++e) {
        const int idx = threadIdx.x + e * 256;
        if (idx < tile && acc[e] != 0.f) atomicAdd(dW + (size_t)k * tile + idx, acc[e]);
    }
}

extern "C" int dz_spconv_wgrad(const float* in, int cin, const int32_t* nbr, int K, int nbr_cap, const int* d_n_out, int out_cap,
                               const float* dout, int cout, float* dW, dz_stream_t stream) {
    DZ_CHECK_ARG(in && nbr && d_n_out && dout && dW && cin >= 1 && cout >= 1 && cin <= 128 && cout <= 128 && K >= 1 && nbr_cap >= out_cap);
    cudaStream_t st = (cudaStream_t)stream;
    DZ_CUDA(cudaMemsetAsync(dW, 0, (size_t)K * cin * cout * sizeof(float), st));
    dim3 grid(dz_cdiv(out_cap, WG_ROWS), K);
    const size_t smem = (size_t)WG_BATCH * (cin + cout) * sizeof(float);
    k_spconv_wgrad<<<grid, 256, smem, st>>>(in, cin, nbr, nbr_cap, d_n_out, out_cap, dout, cout, dW);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

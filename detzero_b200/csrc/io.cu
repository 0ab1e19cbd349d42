// io.cu -- device half of the on-disk frame path (SURVEY.md §8f row 4): a raw Waymo frame file, as the reference writes it
// (detection/detzero_det/datasets/waymo/waymo_utils.py:284-302: (N, 6) float32 [x, y, z, intensity, elongation, NLZ_flag]), goes
// from pinned host memory to the device AS IS; this kernel then does what DatasetTemplate.merge_sweeps does on the host for every
// sweep (detection/detzero_det/datasets/dataset.py:167-196): keep the points with NLZ_flag == -1 (in file order), tanh() the
// intensity, move xyz into the current frame with the 3x4 part of inv(current_pose) @ sweep_pose (double precision like numpy),
// append the sweep's time offset, and -- the collate step (dataset.py:275-283) -- prepend the batch index.  Rows are appended at
// *d_count, so the sweeps of a frame and the frames of a batch concatenate without a host sync.
#include "common.cuh"

struct PrepXform { double m[12]; };           // row-major 3x4

static constexpr int PREP_CHUNK = 1024;

__global__ void __launch_bounds__(256) k_prep_count(const float* __restrict__ raw, int n, int* __restrict__ chunk_counts) {
    const int chunk = blockIdx.x;
    __shared__ int s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    int c = 0;
    for (int p = chunk * PREP_CHUNK + threadIdx.x; p < min(n, (chunk + 1) * PREP_CHUNK); p += 256) c += raw[(size_t)p * 6 + 5] == -1.0f;
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) chunk_counts[chunk] = s_cnt;
}

// exclusive scan of the chunk counts, shifted by the rows already present; bumps *d_count (clamped rows are still counted in
// d_count[1] = rows wanted, so the caller can detect an overflow of `cap`)
__global__ void __launch_bounds__(1024) k_prep_scan(int* __restrict__ chunk_counts, int n_chunks, int* __restrict__ d_count) {
    __shared__ int s_run;
    if (threadIdx.x == 0) s_run = d_count[0];
    __syncthreads();
    for (int base = 0; base < n_chunks; base += 1024) {
        const int k = base + threadIdx.x;
        const int v = k < n_chunks ? chunk_counts[k] : 0;
        int total;
        const int ex = block_exclusive_scan(v, &total);
        if (k < n_chunks) chunk_counts[k] = s_run + ex;
        __syncthreads();
        if (threadIdx.x == 0) s_run += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) { d_count[0] = s_run; d_count[1] = s_run; }
}

__global__ void __launch_bounds__(256) k_prep_write(const float* __restrict__ raw, int n, const int* __restrict__ chunk_base, PrepXform xf,
                                                    int identity, float time_offset, int with_time, float batch_idx, float* __restrict__ out,
                                                    int cap) {
    const int chunk = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __shared__ int s_warp[8];
    const int C = 1 + 5 + (with_time ? 1 : 0);
    int run = chunk_base[chunk];
    for (int p0 = chunk * PREP_CHUNK; p0 < min(n, (chunk + 1) * PREP_CHUNK); p0 += 256) {
        const int p = p0 + threadIdx.x;
        float v[6];
        bool keep = false;
        if (p < n) {
            const float2* q = reinterpret_cast<const float2*>(raw + (size_t)p * 6);
            const float2 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2);
            v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y;
            keep = v[5] == -1.0f;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) { const int cw = s_warp[w]; before += w < warp ? cw : 0; total += cw; }
        if (keep) {
            const int row = run + before + __popc(bal & ((1u << lane) - 1u));
            if (row < cap) {
                float x = v[0], y = v[1], z = v[2];
                if (!identity) {                     // [x y z 1] @ transform[:3, :].T in double, like numpy on a float64 pose
                    const double dx = v[0], dy = v[1], dz = v[2];
                    x = (float)(dx * xf.m[0] + dy * xf.m[1] + dz * xf.m[2] + xf.m[3]);
                    y = (float)(dx * xf.m[4] + dy * xf.m[5] + dz * xf.m[6] + xf.m[7]);
                    z = (float)(dx * xf.m[8] + dy * xf.m[9] + dz * xf.m[10] + xf.m[11]);
                }
                float* o = out + (size_t)row * C;
                o[0] = batch_idx; o[1] = x; o[2] = y; o[3] = z; o[4] = tanhf(v[3]); o[5] = v[4];
                if (with_time) o[6] = time_offset;
            }
        }
        run += total;
        __syncthreads();
    }
}

// the per-chunk counts, scanned in place
static int* carve_prep(DzCarve& cv, int n) { return cv.take<int>(dz_cdiv(max(n, 1), PREP_CHUNK)); }

extern "C" size_t dz_prepare_points_ws_bytes(int n) { return dz_carve_bytes(carve_prep, n); }

extern "C" int dz_prepare_points(const float* raw, int n, const double* transform12_host, float time_offset, int with_time, int batch_idx,
                                 float* out, int cap, int* d_count, void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(raw && out && d_count && n >= 0 && cap >= 1);
    if (n == 0) return DZ_OK;
    DZ_CHECK_WS(dz_prepare_points_ws_bytes(n));
    PrepXform xf;
    int identity = transform12_host == nullptr;
    for (int i = 0; i < 12; ++i) xf.m[i] = identity ? 0.0 : transform12_host[i];
    cudaStream_t st = (cudaStream_t)stream;
    const int n_chunks = dz_cdiv(n, PREP_CHUNK);
    DzCarve cv((char*)ws);
    int* cc = carve_prep(cv, n);
    k_prep_count<<<n_chunks, 256, 0, st>>>(raw, n, cc);
    k_prep_scan<<<1, 1024, 0, st>>>(cc, n_chunks, d_count);
    k_prep_write<<<n_chunks, 256, 0, st>>>(raw, n, cc, xf, identity, time_offset, with_time, (float)batch_idx, out, cap);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// voxelize.cu -- grid-index scan, hard voxelization (+MeanVFE) and dynamic mean voxelization for sm_90a.
//
// Replaces spconv.utils.Point2VoxelCPU3d.point_to_voxel as driven by
// detection/detzero_det/datasets/processor/data_processor.py:61-91, MeanVFE.forward (vfe.py:66-83) and
// DynamicMeanVFE.forward (vfe.py:110-147).
//
// Design (GPU-first, not the CPU algorithm): instead of a sequential dense-grid walk, cells are deduplicated with
// an L2-resident occupancy BITMAP (1 bit/cell, 11.6 MB for the 41x1504x1504 Waymo lattice) that is turned into a
// rank structure by a popcount prefix scan.  "First appearance" order is recovered with atomicMin(first point id)
// per occupied cell + an exclusive scan of leader flags in point order; the first max_pts points of every voxel
// are selected with an order-independent atomicMin cascade.  Point rows are staged through shared memory with
// 128-bit loads; bitmap atomics are warp-aggregated with __match_any_sync.  Every step is deterministic.
//
// The voxel index arithmetic is IEEE fp32 subtract -> divide -> floor (__fsub_rn/__fdiv_rn), never a
// reciprocal multiply or an FMA contraction: see SURVEY.md Appendix A.1.
#include "common.cuh"

#include <cub/device/device_radix_sort.cuh>

#define SENTINEL 0x7f7f7f7f
#define INVALID_CELL 0xffffffffu

// ---------------------------------------------------------------------------------------------------------------
// popcount prefix scan over bitmap words
// ---------------------------------------------------------------------------------------------------------------
static constexpr int SCAN_THREADS = 256;
static constexpr int SCAN_ITEMS = 16;                       // words per thread
static constexpr int SCAN_CHUNK = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ void load_words16(const uint32_t* bm, size_t n_words, size_t base, uint32_t (&w)[SCAN_ITEMS]) {
    if (base + SCAN_ITEMS <= n_words && ((((size_t)(bm + base)) & 15) == 0)) {
        const uint4* p = reinterpret_cast<const uint4*>(bm + base);
#pragma unroll
        for (int j = 0; j < SCAN_ITEMS / 4; ++j) {
            uint4 v = __ldg(p + j);
            w[4 * j] = v.x; w[4 * j + 1] = v.y; w[4 * j + 2] = v.z; w[4 * j + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int j = 0; j < SCAN_ITEMS; ++j) w[j] = (base + j < n_words) ? __ldg(bm + base + j) : 0u;
    }
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_block_sums(const uint32_t* __restrict__ bm, size_t n_words,
                                                                  int* __restrict__ block_sums) {
    size_t base = (size_t)blockIdx.x * SCAN_CHUNK + (size_t)threadIdx.x * SCAN_ITEMS;
    uint32_t w[SCAN_ITEMS];
    load_words16(bm, n_words, base, w);
    int s = 0;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) s += __popc(w[j]);
    int total;
    block_exclusive_scan(s, &total);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// single block: exclusive scan of block_sums in place (+base); *d_total = base + sum
__global__ void __launch_bounds__(1024) k_scan_offsets(int* __restrict__ block_sums, int n_blocks,
                                                       const int* __restrict__ d_base, int* __restrict__ d_total) {
    int carry = d_base ? *d_base : 0;
    for (int start = 0; start < n_blocks; start += 1024) {
        int i = start + threadIdx.x;
        int v = i < n_blocks ? block_sums[i] : 0;
        int tot;
        int ex = block_exclusive_scan(v, &tot);
        if (i < n_blocks) block_sums[i] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0 && d_total) *d_total = carry;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_emit(const uint32_t* __restrict__ bm, uint32_t* __restrict__ prefix,
                                                            size_t n_words, const int* __restrict__ block_offsets) {
    size_t base = (size_t)blockIdx.x * SCAN_CHUNK + (size_t)threadIdx.x * SCAN_ITEMS;
    uint32_t w[SCAN_ITEMS];
    load_words16(bm, n_words, base, w);
    int s = 0;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) s += __popc(w[j]);
    int total;
    int run = block_exclusive_scan(s, &total) + block_offsets[blockIdx.x];
    if (base + SCAN_ITEMS <= n_words && ((((size_t)(prefix + base)) & 15) == 0)) {
        uint4* p = reinterpret_cast<uint4*>(prefix + base);
#pragma unroll
        for (int j = 0; j < SCAN_ITEMS / 4; ++j) {
            uint4 v;
            v.x = run; run += __popc(w[4 * j]);
            v.y = run; run += __popc(w[4 * j + 1]);
            v.z = run; run += __popc(w[4 * j + 2]);
            v.w = run; run += __popc(w[4 * j + 3]);
            p[j] = v;
        }
    } else {
#pragma unroll
        for (int j = 0; j < SCAN_ITEMS; ++j) {
            if (base + j < n_words) prefix[base + j] = run;
            run += __popc(w[j]);
        }
    }
}

static int scan_launch(const uint32_t* bitmap, uint32_t* prefix, size_t n_words, const int* d_base, int* d_total,
                       int* block_sums, cudaStream_t st) {
    int n_blocks = dz_cdiv((long long)n_words, SCAN_CHUNK);
    if (n_blocks == 0) n_blocks = 1;
    k_scan_block_sums<<<n_blocks, SCAN_THREADS, 0, st>>>(bitmap, n_words, block_sums);
    k_scan_offsets<<<1, 1024, 0, st>>>(block_sums, n_blocks, d_base, d_total);
    k_scan_emit<<<n_blocks, SCAN_THREADS, 0, st>>>(bitmap, prefix, n_words, block_sums);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" size_t dz_grid_index_words(int B, int D, int H, int W) {
    return (size_t)((long long)B * dz_cells_pad(D, H, W) / 32);
}

extern "C" size_t dz_scan_ws_bytes(size_t n_words) {
    return dz_align_up((size_t)(dz_cdiv((long long)n_words, SCAN_CHUNK) + 1) * sizeof(int), 256);
}

extern "C" int dz_grid_index_scan(const uint32_t* bitmap, uint32_t* prefix, size_t n_words, const int* d_base,
                                  int* d_total, void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(bitmap && prefix && ws);
    if (ws_bytes < dz_scan_ws_bytes(n_words)) { dz_set_error("dz_grid_index_scan: workspace too small"); return DZ_ERR_WORKSPACE; }
    return scan_launch(bitmap, prefix, n_words, d_base, d_total, (int*)ws, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------------------
// index from an arbitrary coordinate list
// ---------------------------------------------------------------------------------------------------------------
__global__ void k_coords_mark(const int32_t* __restrict__ coords, const int* __restrict__ d_n, int cap, int D, int H, int W,
                              long long cells_pad, uint32_t* __restrict__ bitmap) {
    int n = min(*d_n, cap);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        int4 c = __ldg(reinterpret_cast<const int4*>(coords) + i);   // b,z,y,x
        long long cell = (long long)c.x * cells_pad + ((long long)c.y * H + c.z) * W + c.w;
        atomicOr(bitmap + (cell >> 5), 1u << (cell & 31));
    }
}

__global__ void k_coords_perm(const int32_t* __restrict__ coords, const int* __restrict__ d_n, int cap, int D, int H, int W,
                              long long cells_pad, const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ prefix,
                              int32_t* __restrict__ perm) {
    int n = min(*d_n, cap);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        int4 c = __ldg(reinterpret_cast<const int4*>(coords) + i);
        long long cell = (long long)c.x * cells_pad + ((long long)c.y * H + c.z) * W + c.w;
        size_t w = (size_t)(cell >> 5);
        uint32_t bit = (uint32_t)cell & 31u;
        int rank = (int)(prefix[w] + __popc(bitmap[w] & ((1u << bit) - 1u)));
        perm[rank] = i;
    }
}

extern "C" int dz_grid_index_from_coords(const int32_t* coords, const int* d_n, int cap, int B, int D, int H, int W,
                                         uint32_t* bitmap, uint32_t* prefix, int32_t* perm, int* d_total,
                                         void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(coords && d_n && bitmap && prefix && cap >= 0);
    cudaStream_t st = (cudaStream_t)stream;
    size_t n_words = dz_grid_index_words(B, D, H, W);
    if (ws_bytes < dz_scan_ws_bytes(n_words)) { dz_set_error("dz_grid_index_from_coords: workspace too small"); return DZ_ERR_WORKSPACE; }
    long long cp = dz_cells_pad(D, H, W);
    int blocks = max(1, min(dz_cdiv(cap, 256), DZ_NUM_SMS * 8));
    k_coords_mark<<<blocks, 256, 0, st>>>(coords, d_n, cap, D, H, W, cp, bitmap);
    int rc = scan_launch(bitmap, prefix, n_words, nullptr, d_total, (int*)ws, st);
    if (rc) return rc;
    if (perm) k_coords_perm<<<blocks, 256, 0, st>>>(coords, d_n, cap, D, H, W, cp, bitmap, prefix, perm);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// hard voxelization
// ---------------------------------------------------------------------------------------------------------------
struct VoxGeom {
    float lo[3];      // x,y,z
    float vs[3];      // x,y,z
    int grid[3];      // x,y,z  (valid voxel grid)
    int iD, iH, iW;   // index lattice (z,y,x)
    long long cells_pad;
};

// IEEE fp32: floor((p - lo) / vs).  No FMA, no reciprocal.
__device__ __forceinline__ bool voxel_coord(float p, float lo, float vs, int grid, int& c) {
    float q = floorf(__fdiv_rn(__fsub_rn(p, lo), vs));
    if (!(q >= 0.f && q < (float)grid)) return false;
    c = (int)q;
    return true;
}

static constexpr int VOX_THREADS = 256;

// stage VOX_THREADS rows of `stride` floats through smem with 128-bit loads; returns pointer to this thread's row
template <int MAX_STRIDE>
__device__ __forceinline__ const float* stage_rows(const float* __restrict__ points, int n, int stride, int row0, float* smem) {
    int rows = min(VOX_THREADS, n - row0);
    if (rows <= 0) return smem;
    const float* src = points + (size_t)row0 * stride;
    int nfl = rows * stride;
    if ((((size_t)src) & 15) == 0) {
        int nv = nfl >> 2;
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(smem);
        for (int j = threadIdx.x; j < nv; j += VOX_THREADS) d4[j] = __ldg(s4 + j);
        for (int j = (nv << 2) + threadIdx.x; j < nfl; j += VOX_THREADS) smem[j] = __ldg(src + j);
    } else {
        for (int j = threadIdx.x; j < nfl; j += VOX_THREADS) smem[j] = __ldg(src + j);
    }
    __syncthreads();
    return smem + threadIdx.x * stride;
}

#define VOX_MAX_STRIDE 16

__global__ void __launch_bounds__(VOX_THREADS) k_vox_mark(const float* __restrict__ points, int n, int stride, int xyz_off,
                                                          VoxGeom g, int batch_idx, uint32_t* __restrict__ bitmap,
                                                          uint32_t* __restrict__ cell_out) {
    __shared__ __align__(16) float smem[VOX_THREADS * VOX_MAX_STRIDE];
    int row0 = blockIdx.x * VOX_THREADS;
    const float* row = stage_rows<VOX_MAX_STRIDE>(points, n, stride, row0, smem);
    int i = row0 + threadIdx.x;
    bool valid = false;
    uint32_t cell = INVALID_CELL;
    if (i < n) {
        int cx, cy, cz;
        valid = voxel_coord(row[xyz_off + 0], g.lo[0], g.vs[0], g.grid[0], cx) &&
                voxel_coord(row[xyz_off + 1], g.lo[1], g.vs[1], g.grid[1], cy) &&
                voxel_coord(row[xyz_off + 2], g.lo[2], g.vs[2], g.grid[2], cz);
        if (valid) cell = (uint32_t)((cz * g.iH + cy) * g.iW + cx);
        cell_out[i] = cell;
    }
    unsigned active = __ballot_sync(0xffffffffu, valid);
    if (valid) {
        long long glob = (long long)batch_idx * g.cells_pad + cell;
        unsigned long long w = (unsigned long long)(glob >> 5);
        unsigned bit = 1u << (glob & 31);
        unsigned m = __match_any_sync(active, w);
        unsigned bits = __reduce_or_sync(m, bit);
        if ((threadIdx.x & 31) == __ffs(m) - 1) atomicOr(bitmap + w, bits);
    }
}

__global__ void __launch_bounds__(VOX_THREADS) k_vox_first(const uint32_t* __restrict__ cell, int n, long long cell_base,
                                                           const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ prefix,
                                                           const int* __restrict__ d_counters, int* __restrict__ first_idx,
                                                           uint32_t* __restrict__ rnk) {
    int i = blockIdx.x * VOX_THREADS + threadIdx.x;
    uint32_t c = i < n ? cell[i] : INVALID_CELL;
    bool valid = c != INVALID_CELL;
    unsigned active = __ballot_sync(0xffffffffu, valid);
    if (valid) {
        long long glob = cell_base + c;
        size_t w = (size_t)(glob >> 5);
        uint32_t bit = (uint32_t)glob & 31u;
        int rank = (int)(prefix[w] + __popc(bitmap[w] & ((1u << bit) - 1u))) - d_counters[1];
        rnk[i] = (uint32_t)rank;
        unsigned m = __match_any_sync(active, rank);
        if ((threadIdx.x & 31) == __ffs(m) - 1) atomicMin(first_idx + rank, i);   // lowest lane == lowest point id
    }
}

static constexpr int LEAD_ITEMS = 8;
static constexpr int LEAD_CHUNK = VOX_THREADS * LEAD_ITEMS;

__global__ void __launch_bounds__(VOX_THREADS) k_vox_lead_count(const uint32_t* __restrict__ cell, const uint32_t* __restrict__ rnk,
                                                                const int* __restrict__ first_idx, int n,
                                                                int* __restrict__ block_sums) {
    int base = blockIdx.x * LEAD_CHUNK + threadIdx.x * LEAD_ITEMS;
    int s = 0;
#pragma unroll
    for (int j = 0; j < LEAD_ITEMS; ++j) {
        int i = base + j;
        if (i < n && cell[i] != INVALID_CELL && first_idx[rnk[i]] == i) ++s;
    }
    int tot;
    block_exclusive_scan(s, &tot);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = tot;
}

// emit voxel ids: leader with in-frame rank r < max_voxels gets row vid_base + r
__global__ void __launch_bounds__(VOX_THREADS) k_vox_lead_emit(const uint32_t* __restrict__ cell, const uint32_t* __restrict__ rnk,
                                                               const int* __restrict__ first_idx, int n,
                                                               const int* __restrict__ block_offsets, VoxGeom g, int batch_idx,
                                                               int max_voxels, int cap, const int* __restrict__ d_counters,
                                                               int32_t* __restrict__ coords, int32_t* __restrict__ perm) {
    int base = blockIdx.x * LEAD_CHUNK + threadIdx.x * LEAD_ITEMS;
    bool lead[LEAD_ITEMS];
    int s = 0;
#pragma unroll
    for (int j = 0; j < LEAD_ITEMS; ++j) {
        int i = base + j;
        lead[j] = (i < n && cell[i] != INVALID_CELL && first_idx[rnk[i]] == i);
        s += lead[j];
    }
    int tot;
    int r = block_exclusive_scan(s, &tot) + block_offsets[blockIdx.x];
    const int vid_base = d_counters[0], rank_base = d_counters[1];
#pragma unroll
    for (int j = 0; j < LEAD_ITEMS; ++j) {
        if (!lead[j]) continue;
        int i = base + j;
        int vid = -1;
        if (r < max_voxels && vid_base + r < cap) {
            vid = vid_base + r;
            uint32_t c = cell[i];
            int cx = c % g.iW, t = c / g.iW;
            int cy = t % g.iH, cz = t / g.iH;
            reinterpret_cast<int4*>(coords)[vid] = make_int4(batch_idx, cz, cy, cx);
        }
        perm[rank_base + rnk[i]] = vid;
        ++r;
    }
}

// keep the max_pts smallest point ids per voxel: order-independent atomicMin cascade (lists[p*L + v])
__global__ void __launch_bounds__(VOX_THREADS) k_vox_slots(const uint32_t* __restrict__ cell, const uint32_t* __restrict__ rnk, int n,
                                                           const int32_t* __restrict__ perm, const int* __restrict__ d_counters,
                                                           int max_pts, int L, int* __restrict__ lists) {
    int i = blockIdx.x * VOX_THREADS + threadIdx.x;
    if (i >= n || cell[i] == INVALID_CELL) return;
    int vid = perm[d_counters[1] + rnk[i]];
    if (vid < 0) return;
    int v = vid - d_counters[0];
    if (lists[(size_t)(max_pts - 1) * L + v] < i) return;      // already max_pts smaller ids (values only decrease)
    int val = i;
    for (int p = 0; p < max_pts; ++p) {
        int old = atomicMin(lists + (size_t)p * L + v, val);
        if (old > val) val = old;                                // we placed ours; carry the displaced one
        if (val == SENTINEL) break;
    }
}

__global__ void __launch_bounds__(VOX_THREADS) k_vox_write(const float* __restrict__ points, int stride, int feat_off, int c,
                                                           const int* __restrict__ lists, int L, int max_pts, int max_voxels,
                                                           int cap, const int* __restrict__ d_tmp, const int* __restrict__ d_counters,
                                                           float* __restrict__ voxels, int32_t* __restrict__ num_per,
                                                           float* __restrict__ mean) {
    int n_vox = min(d_tmp[1], max_voxels);
    int vid_base = d_counters[0];
    n_vox = min(n_vox, cap - vid_base);
    int v = blockIdx.x * VOX_THREADS + threadIdx.x;
    if (v >= n_vox) return;
    size_t vid = (size_t)vid_base + v;
    float sum[VOX_MAX_STRIDE];
    for (int k = 0; k < c; ++k) sum[k] = 0.f;
    int cnt = 0;
    for (int p = 0; p < max_pts; ++p) {
        int idx = lists[(size_t)p * L + v];
        float* dst = voxels + (vid * max_pts + p) * c;
        if (idx != SENTINEL) {
            const float* src = points + (size_t)idx * stride + feat_off;
            for (int k = 0; k < c; ++k) { float f = __ldg(src + k); dst[k] = f; sum[k] += f; }
            ++cnt;
        } else {
            for (int k = 0; k < c; ++k) dst[k] = 0.f;
        }
    }
    num_per[vid] = cnt;
    if (mean) {
        float denom = (float)max(cnt, 1);                        // clamp_min(num, 1.0), vfe.py:79-80
        for (int k = 0; k < c; ++k) mean[vid * c + k] = __fdiv_rn(sum[k], denom);
    }
}

__global__ void k_vox_finish(const int* __restrict__ d_tmp, int max_voxels, int cap, int* __restrict__ d_counters) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        int want = min(d_tmp[1], max_voxels);
        int nv = min(want, cap - d_counters[0]);
        d_counters[0] += nv;
        d_counters[1] = d_tmp[0];
        d_counters[2] += want;          // rows the caller's capacity should have held (== [0] unless cap was too small)
    }
}

// scan of the leader block sums (single block) writing the total into d_tmp[1]
extern "C" size_t dz_voxelize_hard_ws_bytes(int n_points, int max_pts, int max_voxels, int iD, int iH, int iW) {
    size_t n = (size_t)(n_points > 0 ? n_points : 1);
    size_t L = (size_t)(n_points < max_voxels ? (n_points > 0 ? n_points : 1) : max_voxels);
    size_t frame_words = (size_t)(dz_cells_pad(iD, iH, iW) / 32);
    size_t b = 0;
    b += dz_align_up(n * 4, 256) * 3;                            // cell, rnk, first_idx
    b += dz_align_up(L * max_pts * 4, 256);                      // lists
    b += dz_scan_ws_bytes(frame_words);                          // bitmap scan block sums
    b += dz_align_up((size_t)(dz_cdiv((long long)n, LEAD_CHUNK) + 1) * 4, 256);
    b += 256;                                                    // tmp ints
    return b;
}

extern "C" int dz_voxelize_hard(const float* points, int n, int point_stride, int xyz_off, int c,
                                const float* range6, const float* vsize3, const int* grid_zyx3,
                                int max_pts, int max_voxels, int batch_idx,
                                float* voxels, int32_t* coords, int32_t* num_per_voxel, float* mean, int cap,
                                int* d_counters, int B, int iD, int iH, int iW, uint32_t* index_bitmap,
                                uint32_t* index_prefix, int32_t* index_perm, void* ws, size_t ws_bytes,
                                dz_stream_t stream) {
    DZ_CHECK_ARG((points || n == 0) && voxels && coords && num_per_voxel && d_counters && index_bitmap && index_prefix && index_perm);
    DZ_CHECK_ARG(n >= 0 && c >= 1 && xyz_off >= 0 && xyz_off + c <= point_stride && point_stride <= VOX_MAX_STRIDE && c >= 3);
    DZ_CHECK_ARG(max_pts >= 1 && max_voxels >= 1 && batch_idx >= 0 && batch_idx < B);
    DZ_CHECK_ARG(grid_zyx3[0] <= iD && grid_zyx3[1] <= iH && grid_zyx3[2] <= iW);
    if (ws_bytes < dz_voxelize_hard_ws_bytes(n, max_pts, max_voxels, iD, iH, iW)) {
        dz_set_error("dz_voxelize_hard: workspace too small"); return DZ_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    VoxGeom g;
    for (int d = 0; d < 3; ++d) { g.lo[d] = range6[d]; g.vs[d] = vsize3[d]; g.grid[d] = grid_zyx3[2 - d]; }
    g.iD = iD; g.iH = iH; g.iW = iW; g.cells_pad = dz_cells_pad(iD, iH, iW);
    size_t frame_words = (size_t)(g.cells_pad / 32);
    size_t nn = (size_t)(n > 0 ? n : 1);
    int L = n < max_voxels ? (n > 0 ? n : 1) : max_voxels;

    DzWs w(ws, ws_bytes);
    uint32_t* cell = w.take<uint32_t>(nn);
    uint32_t* rnk = w.take<uint32_t>(nn);
    int* first_idx = w.take<int>(nn);
    int* lists = w.take<int>((size_t)L * max_pts);
    int* scan_sums = (int*)w.take<char>(dz_scan_ws_bytes(frame_words));
    int n_lead_blocks = max(1, dz_cdiv(n, LEAD_CHUNK));
    int* lead_sums = w.take<int>(n_lead_blocks + 1);
    int* d_tmp = w.take<int>(4);
    if (!d_tmp) { dz_set_error("dz_voxelize_hard: workspace carve failed"); return DZ_ERR_WORKSPACE; }

    DZ_CUDA(cudaMemsetAsync(first_idx, 0x7f, nn * 4, st));
    DZ_CUDA(cudaMemsetAsync(lists, 0x7f, (size_t)L * max_pts * 4, st));
    int pblocks = max(1, dz_cdiv(n, VOX_THREADS));
    uint32_t* bm_frame = index_bitmap + (size_t)batch_idx * frame_words;
    uint32_t* pf_frame = index_prefix + (size_t)batch_idx * frame_words;

    k_vox_mark<<<pblocks, VOX_THREADS, 0, st>>>(points, n, point_stride, xyz_off, g, batch_idx, index_bitmap, cell);
    // prefix of this frame's words, continuing the rank count of previous frames (d_counters[1])
    int rc = scan_launch(bm_frame, pf_frame, frame_words, d_counters + 1, d_tmp + 0, scan_sums, st);
    if (rc) return rc;
    k_vox_first<<<pblocks, VOX_THREADS, 0, st>>>(cell, n, (long long)batch_idx * g.cells_pad, index_bitmap, index_prefix,
                                                 d_counters, first_idx, rnk);
    k_vox_lead_count<<<n_lead_blocks, VOX_THREADS, 0, st>>>(cell, rnk, first_idx, n, lead_sums);
    k_scan_offsets<<<1, 1024, 0, st>>>(lead_sums, n_lead_blocks, nullptr, d_tmp + 1);
    k_vox_lead_emit<<<n_lead_blocks, VOX_THREADS, 0, st>>>(cell, rnk, first_idx, n, lead_sums, g, batch_idx, max_voxels, cap,
                                                           d_counters, coords, index_perm);
    k_vox_slots<<<pblocks, VOX_THREADS, 0, st>>>(cell, rnk, n, index_perm, d_counters, max_pts, L, lists);
    k_vox_write<<<max(1, dz_cdiv(L, VOX_THREADS)), VOX_THREADS, 0, st>>>(points, point_stride, xyz_off, c, lists, L, max_pts,
                                                                         max_voxels, cap, d_tmp, d_counters, voxels,
                                                                         num_per_voxel, mean);
    k_vox_finish<<<1, 32, 0, st>>>(d_tmp, max_voxels, cap, d_counters);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Batched hard voxelization: the frames of a batch are independent except for two running totals (occupied cells ->
// rank base, emitted voxels -> row base).  Each frame runs on its own internal stream; a frame only waits for its
// predecessor's bitmap scan (rank base) and leader scan (row base), so the ~10 latency-bound kernels of the 8 frames of a
// batch overlap instead of running back to back.  Forked from / joined to the caller's stream with events (capturable in a
// CUDA graph).  Results are identical to B calls of dz_voxelize_hard in frame order.
// ---------------------------------------------------------------------------------------------------------------
static constexpr int VB_STREAMS = 8, VB_MAX_FRAMES = 256;
struct VbPool {
    bool init = false;
    cudaStream_t s[VB_STREAMS];
    cudaEvent_t fork, done[VB_STREAMS], rank_ev[VB_MAX_FRAMES], vid_ev[VB_MAX_FRAMES];
};
static VbPool g_vb;

__global__ void k_vb_pub_rank(const int* __restrict__ d_tmp, int* __restrict__ ctr_next) {
    if (threadIdx.x == 0) ctr_next[1] = d_tmp[0];                 // occupied cells up to and including this frame
}
__global__ void k_vb_pub_vid(const int* __restrict__ d_tmp, const int* __restrict__ ctr, int max_voxels, int cap, int* __restrict__ ctr_next) {
    if (threadIdx.x == 0) {
        int want = min(d_tmp[1], max_voxels);
        int nv = min(want, cap - ctr[0]);
        ctr_next[0] = ctr[0] + nv;
        ctr_next[2] = ctr[2] + want;          // rows the caller's capacity should have held
    }
}

extern "C" size_t dz_voxelize_hard_batch_ws_bytes(int n_max, int B, int max_pts, int max_voxels, int iD, int iH, int iW) {
    return (size_t)B * dz_align_up(dz_voxelize_hard_ws_bytes(n_max, max_pts, max_voxels, iD, iH, iW), 256) + dz_align_up((size_t)(B + 1) * 16, 256);
}

extern "C" int dz_voxelize_hard_batch(const float* const* points_host, const int* n_host, int B, int point_stride, int xyz_off, int c,
                                      const float* range6, const float* vsize3, const int* grid_zyx3, int max_pts, int max_voxels,
                                      float* voxels, int32_t* coords, int32_t* num_per_voxel, float* mean, int cap, int* d_counters,
                                      int iD, int iH, int iW, uint32_t* index_bitmap, uint32_t* index_prefix, int32_t* index_perm,
                                      void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(points_host && n_host && voxels && coords && num_per_voxel && d_counters && index_bitmap && index_prefix && index_perm);
    DZ_CHECK_ARG(B >= 1 && B <= VB_MAX_FRAMES && c >= 3 && xyz_off >= 0 && xyz_off + c <= point_stride && point_stride <= VOX_MAX_STRIDE);
    DZ_CHECK_ARG(max_pts >= 1 && max_voxels >= 1 && grid_zyx3[0] <= iD && grid_zyx3[1] <= iH && grid_zyx3[2] <= iW);
    int n_max = 0;
    for (int b = 0; b < B; ++b) { DZ_CHECK_ARG(n_host[b] >= 0 && (points_host[b] || n_host[b] == 0)); n_max = max(n_max, n_host[b]); }
    if (ws_bytes < dz_voxelize_hard_batch_ws_bytes(n_max, B, max_pts, max_voxels, iD, iH, iW)) {
        dz_set_error("dz_voxelize_hard_batch: workspace too small"); return DZ_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (!g_vb.init) {
        for (int i = 0; i < VB_STREAMS; ++i) {
            DZ_CUDA(cudaStreamCreateWithFlags(&g_vb.s[i], cudaStreamNonBlocking));
            DZ_CUDA(cudaEventCreateWithFlags(&g_vb.done[i], cudaEventDisableTiming));
        }
        DZ_CUDA(cudaEventCreateWithFlags(&g_vb.fork, cudaEventDisableTiming));
        for (int i = 0; i < VB_MAX_FRAMES; ++i) {
            DZ_CUDA(cudaEventCreateWithFlags(&g_vb.rank_ev[i], cudaEventDisableTiming));
            DZ_CUDA(cudaEventCreateWithFlags(&g_vb.vid_ev[i], cudaEventDisableTiming));
        }
        g_vb.init = true;
    }
    VoxGeom g;
    for (int d = 0; d < 3; ++d) { g.lo[d] = range6[d]; g.vs[d] = vsize3[d]; g.grid[d] = grid_zyx3[2 - d]; }
    g.iD = iD; g.iH = iH; g.iW = iW; g.cells_pad = dz_cells_pad(iD, iH, iW);
    const size_t frame_words = (size_t)(g.cells_pad / 32);
    const size_t per_frame = dz_align_up(dz_voxelize_hard_ws_bytes(n_max, max_pts, max_voxels, iD, iH, iW), 256);
    unsigned char* wsb = reinterpret_cast<unsigned char*>(ws);
    int* ctr = reinterpret_cast<int*>(wsb + (size_t)B * per_frame);          // (B+1) x {row base, rank base, rows wanted, pad}
    DZ_CUDA(cudaMemcpyAsync(ctr, d_counters, 12, cudaMemcpyDeviceToDevice, st));
    DZ_CUDA(cudaEventRecord(g_vb.fork, st));
    const int S = min(B, VB_STREAMS);
    for (int i = 0; i < S; ++i) DZ_CUDA(cudaStreamWaitEvent(g_vb.s[i], g_vb.fork, 0));
    for (int b = 0; b < B; ++b) {
        cudaStream_t s = g_vb.s[b % S];
        const float* points = points_host[b];
        const int n = n_host[b];
        const size_t nn = (size_t)(n > 0 ? n : 1);
        const int L = n < max_voxels ? (n > 0 ? n : 1) : max_voxels;
        DzWs w(wsb + (size_t)b * per_frame, per_frame);
        uint32_t* cell = w.take<uint32_t>(nn);
        uint32_t* rnk = w.take<uint32_t>(nn);
        int* first_idx = w.take<int>(nn);
        int* lists = w.take<int>((size_t)L * max_pts);
        int* scan_sums = (int*)w.take<char>(dz_scan_ws_bytes(frame_words));
        const int n_lead_blocks = max(1, dz_cdiv(n, LEAD_CHUNK));
        int* lead_sums = w.take<int>(n_lead_blocks + 1);
        int* d_tmp = w.take<int>(4);
        if (!d_tmp) { dz_set_error("dz_voxelize_hard_batch: workspace carve failed"); return DZ_ERR_WORKSPACE; }
        int* ctr_b = ctr + 4 * b;
        int* ctr_n = ctr + 4 * (b + 1);
        DZ_CUDA(cudaMemsetAsync(first_idx, 0x7f, nn * 4, s));
        DZ_CUDA(cudaMemsetAsync(lists, 0x7f, (size_t)L * max_pts * 4, s));
        const int pblocks = max(1, dz_cdiv(n, VOX_THREADS));
        uint32_t* bm_frame = index_bitmap + (size_t)b * frame_words;
        uint32_t* pf_frame = index_prefix + (size_t)b * frame_words;
        k_vox_mark<<<pblocks, VOX_THREADS, 0, s>>>(points, n, point_stride, xyz_off, g, b, index_bitmap, cell);
        if (b > 0) DZ_CUDA(cudaStreamWaitEvent(s, g_vb.rank_ev[b - 1], 0));       // ctr_b[1] = cells of the frames before
        int rc = scan_launch(bm_frame, pf_frame, frame_words, ctr_b + 1, d_tmp + 0, scan_sums, s);
        if (rc) return rc;
        k_vb_pub_rank<<<1, 32, 0, s>>>(d_tmp, ctr_n);
        DZ_CUDA(cudaEventRecord(g_vb.rank_ev[b], s));
        k_vox_first<<<pblocks, VOX_THREADS, 0, s>>>(cell, n, (long long)b * g.cells_pad, index_bitmap, index_prefix, ctr_b, first_idx, rnk);
        k_vox_lead_count<<<n_lead_blocks, VOX_THREADS, 0, s>>>(cell, rnk, first_idx, n, lead_sums);
        k_scan_offsets<<<1, 1024, 0, s>>>(lead_sums, n_lead_blocks, nullptr, d_tmp + 1);
        if (b > 0) DZ_CUDA(cudaStreamWaitEvent(s, g_vb.vid_ev[b - 1], 0));        // ctr_b[0], ctr_b[2] = rows of the frames before
        k_vb_pub_vid<<<1, 32, 0, s>>>(d_tmp, ctr_b, max_voxels, cap, ctr_n);
        DZ_CUDA(cudaEventRecord(g_vb.vid_ev[b], s));
        k_vox_lead_emit<<<n_lead_blocks, VOX_THREADS, 0, s>>>(cell, rnk, first_idx, n, lead_sums, g, b, max_voxels, cap, ctr_b, coords, index_perm);
        k_vox_slots<<<pblocks, VOX_THREADS, 0, s>>>(cell, rnk, n, index_perm, ctr_b, max_pts, L, lists);
        k_vox_write<<<max(1, dz_cdiv(L, VOX_THREADS)), VOX_THREADS, 0, s>>>(points, point_stride, xyz_off, c, lists, L, max_pts, max_voxels, cap,
                                                                           d_tmp, ctr_b, voxels, num_per_voxel, mean);
    }
    for (int i = 0; i < S; ++i) {
        DZ_CUDA(cudaEventRecord(g_vb.done[i], g_vb.s[i]));
        DZ_CUDA(cudaStreamWaitEvent(st, g_vb.done[i], 0));
    }
    DZ_CUDA(cudaMemcpyAsync(d_counters, ctr + 4 * B, 12, cudaMemcpyDeviceToDevice, st));
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// MeanVFE.forward on already-voxelized input (vfe.py:66-83): mean over the first num points of each voxel
__global__ void k_mean_vfe(const float* __restrict__ voxels, const int32_t* __restrict__ num, int M, int P, int C,
                           float* __restrict__ out) {
    long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= (long long)M * C) return;
    int v = (int)(t / C), c = (int)(t % C);
    float s = 0.f;
    for (int p = 0; p < P; ++p) s += __ldg(voxels + ((size_t)v * P + p) * C + c);      // sum(dim=1) over all P slots
    out[t] = __fdiv_rn(s, (float)max(num[v], 1));
}

extern "C" int dz_mean_vfe(const float* voxels, const int32_t* num_per_voxel, int M, int P, int C, float* out,
                           dz_stream_t stream) {
    DZ_CHECK_ARG(voxels && num_per_voxel && out && M >= 0 && P >= 1 && C >= 1);
    if (M == 0) return DZ_OK;
    k_mean_vfe<<<dz_cdiv((long long)M * C, 256), 256, 0, (cudaStream_t)stream>>>(voxels, num_per_voxel, M, P, C, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// dynamic mean voxelization (DynamicMeanVFE, vfe.py:110-147)
// ---------------------------------------------------------------------------------------------------------------
struct DynGeom {
    float lo[3], vs[3];
    int grid[3];              // x,y,z
    long long cells_pad;      // round_up(X*Y*Z, 32)
};

__global__ void __launch_bounds__(VOX_THREADS) k_dyn_mark(const float* __restrict__ points, int n, int stride, DynGeom g, int B,
                                                          uint32_t* __restrict__ bitmap, long long* __restrict__ cell_out) {
    __shared__ __align__(16) float smem[VOX_THREADS * VOX_MAX_STRIDE];
    int row0 = blockIdx.x * VOX_THREADS;
    const float* row = stage_rows<VOX_MAX_STRIDE>(points, n, stride, row0, smem);
    int i = row0 + threadIdx.x;
    if (i >= n) return;
    int cx, cy, cz;
    bool valid = voxel_coord(row[1], g.lo[0], g.vs[0], g.grid[0], cx) &&
                 voxel_coord(row[2], g.lo[1], g.vs[1], g.grid[1], cy) &&
                 voxel_coord(row[3], g.lo[2], g.vs[2], g.grid[2], cz);
    int b = (int)row[0];                                        // points[:,0].int()
    valid = valid && b >= 0 && b < B;
    long long cell = -1;
    if (valid) {
        // key order of vfe.py:128-131: b*XYZ + x*YZ + y*Z + z
        cell = (long long)b * g.cells_pad + ((long long)cx * g.grid[1] + cy) * g.grid[2] + cz;
        atomicOr(bitmap + (cell >> 5), 1u << (cell & 31));
    }
    cell_out[i] = cell;
}

// sort key of every point: its voxel's rank (ranks ascend with the b,x,y,z key), n for a dropped point
__global__ void __launch_bounds__(VOX_THREADS) k_dyn_key(const long long* __restrict__ cell_in, int n,
                                                         const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ prefix,
                                                         uint32_t* __restrict__ key, int* __restrict__ idx) {
    int i = blockIdx.x * VOX_THREADS + threadIdx.x;
    if (i >= n) return;
    long long cell = cell_in[i];
    uint32_t k = (uint32_t)n;
    if (cell >= 0) {
        size_t w = (size_t)(cell >> 5);
        uint32_t bit = (uint32_t)cell & 31u;
        k = prefix[w] + __popc(bitmap[w] & ((1u << bit) - 1u));
    }
    key[i] = k;
    idx[i] = i;
}

// after the stable sort by rank: every voxel's points form one run [beg, end) in ascending point index
__global__ void __launch_bounds__(VOX_THREADS) k_dyn_runs(const uint32_t* __restrict__ key, const int* __restrict__ idx, int n,
                                                          const long long* __restrict__ cell_in, DynGeom g, const int* __restrict__ d_m,
                                                          int cap, int* __restrict__ beg, int* __restrict__ end,
                                                          int32_t* __restrict__ coords) {
    int j = blockIdx.x * VOX_THREADS + threadIdx.x;
    if (j >= n) return;
    uint32_t k = key[j];
    if (k >= (uint32_t)min(*d_m, cap)) return;                  // dropped point, or a voxel beyond the caller's capacity
    if (j == 0 || key[j - 1] != k) {
        beg[k] = j;
        long long cell = cell_in[idx[j]];
        long long b = cell / g.cells_pad, r = cell % g.cells_pad;
        int cz = (int)(r % g.grid[2]); r /= g.grid[2];
        int cy = (int)(r % g.grid[1]);
        int cx = (int)(r / g.grid[1]);
        reinterpret_cast<int4*>(coords)[k] = make_int4((int)b, cz, cy, cx);     // [b,z,y,x], vfe.py:143
    }
    if (j == n - 1 || key[j + 1] != k) end[k] = j + 1;
}

// mean of every voxel column: one fp32 sum in ascending point index, then an IEEE divide by the count (torch_scatter's
// scatter_mean on the CPU).  Rows m..cap-1 are zeroed.
__global__ void k_dyn_mean(const float* __restrict__ points, int stride, int c, const int* __restrict__ idx,
                           const int* __restrict__ beg, const int* __restrict__ end, const int* __restrict__ d_m, int cap,
                           float* __restrict__ feats) {
    int m = min(*d_m, cap);
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < (long long)cap * c; t += (long long)gridDim.x * blockDim.x) {
        int r = (int)(t / c), k = (int)(t % c);
        float s = 0.f;
        if (r < m) {
            int j0 = beg[r], j1 = end[r];
#pragma unroll 4
            for (int j = j0; j < j1; ++j) s = __fadd_rn(s, __ldg(points + (size_t)__ldg(idx + j) * stride + 1 + k));
            s = __fdiv_rn(s, (float)(j1 - j0));
        }
        feats[t] = s;
    }
}

static int dyn_key_bits(int n) { return n > 0 ? 32 - __builtin_clz((unsigned)n) : 1; }   // keys are 0..n

static size_t dyn_sort_bytes(int n) {
    size_t bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int*)nullptr, (int*)nullptr,
                                        n, 0, dyn_key_bits(n)) != cudaSuccess)
        return 0;
    return bytes;
}

extern "C" size_t dz_voxelize_dynamic_ws_bytes(int n_points, int cap, int B, int X, int Y, int Z) {
    size_t words = (size_t)((long long)B * dz_cells_pad(X, Y, Z) / 32);
    size_t n = (size_t)(n_points > 0 ? n_points : 1);
    return dz_align_up(words * 4, 256) * 2 + dz_align_up(n * 8, 256) + dz_align_up(n * 4, 256) * 4 +
           dz_align_up((size_t)cap * 4, 256) * 2 + dz_align_up(dyn_sort_bytes(n_points > 0 ? n_points : 0), 256) +
           dz_scan_ws_bytes(words) + 256;
}

// Every voxel's mean is summed in ascending point index, so the result does not depend on launch timing: the same frame gives
// the same bits on every run and under CUDA-graph replay, equal to the reference's sequential scatter on the CPU.  Points are
// stable-sorted by voxel rank (CUB radix sort over the bits of 0..n), then one thread per voxel column walks its run.
extern "C" int dz_voxelize_dynamic_mean(const float* points, int n, int c, int B, const float* range6, const float* vsize3,
                                        const int* grid_xyz3, float* feats, int32_t* coords, int cap, int* d_m,
                                        void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG((points || n == 0) && feats && coords && d_m && n >= 0 && c >= 3 && 1 + c <= VOX_MAX_STRIDE && B >= 1 && cap >= 1);
    if (ws_bytes < dz_voxelize_dynamic_ws_bytes(n, cap, B, grid_xyz3[0], grid_xyz3[1], grid_xyz3[2])) {
        dz_set_error("dz_voxelize_dynamic_mean: workspace too small"); return DZ_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    DynGeom g;
    for (int d = 0; d < 3; ++d) { g.lo[d] = range6[d]; g.vs[d] = vsize3[d]; g.grid[d] = grid_xyz3[d]; }
    g.cells_pad = dz_cells_pad(g.grid[0], g.grid[1], g.grid[2]);
    size_t words = (size_t)((long long)B * g.cells_pad / 32);
    size_t nn = (size_t)(n > 0 ? n : 1);
    size_t sort_bytes = dyn_sort_bytes(n);
    DzWs w(ws, ws_bytes);
    uint32_t* bitmap = w.take<uint32_t>(words);
    uint32_t* prefix = w.take<uint32_t>(words);
    long long* cell = w.take<long long>(nn);
    uint32_t* key = w.take<uint32_t>(nn);
    uint32_t* key_sorted = w.take<uint32_t>(nn);
    int* idx = w.take<int>(nn);
    int* idx_sorted = w.take<int>(nn);
    int* beg = w.take<int>(cap);
    int* end = w.take<int>(cap);
    void* sort_tmp = w.take<char>(sort_bytes > 0 ? sort_bytes : 1);
    int* sums = (int*)w.take<char>(dz_scan_ws_bytes(words));
    if (!sums) { dz_set_error("dz_voxelize_dynamic_mean: workspace carve failed"); return DZ_ERR_WORKSPACE; }
    DZ_CUDA(cudaMemsetAsync(bitmap, 0, words * 4, st));
    int pblocks = max(1, dz_cdiv(n, VOX_THREADS));
    k_dyn_mark<<<pblocks, VOX_THREADS, 0, st>>>(points, n, 1 + c, g, B, bitmap, cell);
    int rc = scan_launch(bitmap, prefix, words, nullptr, d_m, sums, st);
    if (rc) return rc;
    if (n > 0) {
        k_dyn_key<<<pblocks, VOX_THREADS, 0, st>>>(cell, n, bitmap, prefix, key, idx);
        DZ_CUDA(cub::DeviceRadixSort::SortPairs(sort_tmp, sort_bytes, key, key_sorted, idx, idx_sorted, n, 0, dyn_key_bits(n), st));
        k_dyn_runs<<<pblocks, VOX_THREADS, 0, st>>>(key_sorted, idx_sorted, n, cell, g, d_m, cap, beg, end, coords);
    }
    k_dyn_mean<<<DZ_NUM_SMS * 4, 256, 0, st>>>(points, 1 + c, c, idx_sorted, beg, end, d_m, cap, feats);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

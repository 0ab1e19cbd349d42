// combine.cu -- the last DetZero stage on the device: the refined tracks of one sequence (PRM boxes, GRM size, CRM or tracker
// score) and, optionally, the tracker's dropped detections, written as per-frame result rows.  Replaces convert_frame_format and
// combine_det as combine_final drives them (daemon/combine_output.py:27-41,44-99,102-167).
//
// Row of a track box: the PRM lidar box cast to float32 with dx, dy, dz replaced by the GRM prediction's size (combine_final
// :126-129; the reference reads the size from the GRM's reverted lidar boxes, and the revert copies it unchanged, so the prediction
// gives the same bits), the given score (CRM pred_score or the tracker's, :130-131), the track's class as the label.
// Row order in a frame (order_map, :54-59): track rows first, by track, each track's rows in its box order; then the frame's
// dropped detections in input-row order (combine_det), their heading wrapped as the tracker's det_drop wraps it.
// A frame with no track row gets no row at all, not even a dropped one: combine_det only extends frames convert_frame_format emitted.
//
// Deterministic: no atomic decides a row's position.  k_combine_count counts each track's boxes per frame and each box's rank among
// its track's boxes in the same frame; k_combine_frame scans those counts along the tracks for each frame and writes the dropped
// rows; k_combine_write puts each track box at its frame offset + rank.  Nothing assumes a track's frames are ordered or distinct.
// Past R rows in a frame nothing is written out of bounds, count[f] is clamped to R and overflow bit 1 is set; a frame index
// outside 0..F-1 sets bit 2 and its box is skipped.
#include "common.cuh"

namespace {

constexpr int NT = 256;

__device__ __forceinline__ float yaw_filter(float y) {           // track.py _yaw_filter, float32 steps without contraction
    const float pi2 = (float)(3.141592653589793 * 2.0), pi = (float)3.141592653589793;
    if (fabsf(y) >= pi2) y = __fsub_rn(y, __fmul_rn(floorf(__fdiv_rn(y, pi2)), pi2));
    if (y > pi) y = __fsub_rn(y, pi2);
    if (y <= -pi) y = __fadd_rn(y, pi2);
    return y;
}

// one block per track: rank of each box among the track's boxes of the same frame; the first of them stores the count
__global__ void __launch_bounds__(NT) k_combine_count(const int32_t* __restrict__ fob, const int32_t* __restrict__ box_num, int B,
                                                      int L, int F, int32_t* __restrict__ cnt, int32_t* __restrict__ rank,
                                                      int32_t* __restrict__ overflow) {
    const int b = blockIdx.x;
    const int n = min(max(box_num[b], 0), L);
    const int32_t* fb = fob + (size_t)b * L;
    for (int j = threadIdx.x; j < n; j += NT) {
        const int f = fb[j];
        if (f < 0 || f >= F) { atomicOr(overflow, 2); continue; }
        int r = 0;
        for (int i = 0; i < j; ++i) r += fb[i] == f;
        rank[(size_t)b * L + j] = r;
        if (r == 0) {
            int c = 1;
            for (int i = j + 1; i < n; ++i) c += fb[i] == f;
            cnt[(size_t)f * B + b] = c;
        }
    }
}

// block-wide exclusive scan of one value per thread; returns the exclusive prefix, *total the block sum
__device__ int block_scan(int v, int* total) {
    __shared__ int warp_sum[NT / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sum[w] = x;
    __syncthreads();
    if (w == 0) {
        int s = lane < NT / 32 ? warp_sum[lane] : 0;
        for (int o = 1; o < NT / 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        if (lane < NT / 32) warp_sum[lane] = s;                   // inclusive over warps
    }
    __syncthreads();
    const int before = w ? warp_sum[w - 1] : 0;
    *total = warp_sum[NT / 32 - 1];
    __syncthreads();                                              // warp_sum is reused by the next call
    return before + x - v;
}

// one block per frame: offsets of each track's rows (in place in cnt), the frame's dropped rows, its count and overflow
__global__ void __launch_bounds__(NT) k_combine_frame(int32_t* __restrict__ cnt, int B, const float* __restrict__ det,
                                                      const int32_t* __restrict__ det_count, const unsigned char* __restrict__ kept,
                                                      int K, int R, float* __restrict__ rows, int32_t* __restrict__ obj_id,
                                                      int32_t* __restrict__ count, int32_t* __restrict__ overflow) {
    const int f = blockIdx.x;
    int32_t* c = cnt + (size_t)f * B;
    int carry = 0;
    for (int b0 = 0; b0 < B; b0 += NT) {
        const int b = b0 + threadIdx.x;
        const int v = b < B ? c[b] : 0;
        int tot;
        const int ex = block_scan(v, &tot);
        if (b < B) c[b] = carry + ex;
        carry += tot;
    }
    const int tracks = carry;
    int total = tracks;
    if (tracks > 0 && det) {
        const int n = min(max(det_count[f], 0), K);
        for (int k0 = 0; k0 < n; k0 += NT) {
            const int k = k0 + threadIdx.x;
            const int d = k < n && !kept[(size_t)f * K + k];
            int tot;
            const int pos = total + block_scan(d, &tot);
            if (d && pos < R) {
                const float* src = det + ((size_t)f * K + k) * 9;
                float* dst = rows + ((size_t)f * R + pos) * 9;
                for (int i = 0; i < 6; ++i) dst[i] = src[i];
                dst[6] = yaw_filter(src[6]);
                dst[7] = src[7];
                dst[8] = src[8];
                obj_id[(size_t)f * R + pos] = -1;
            }
            total += tot;
        }
    }
    if (threadIdx.x == 0) {
        count[f] = min(total, R);
        if (total > R) atomicOr(overflow, 1);
    }
}

// one block per track: each box's row at its frame's offset for the track + its rank
__global__ void __launch_bounds__(NT) k_combine_write(const double* __restrict__ prm, const float* __restrict__ grm,
                                                      const float* __restrict__ score, const int32_t* __restrict__ fob,
                                                      const int32_t* __restrict__ box_num, const int32_t* __restrict__ cls,
                                                      const int32_t* __restrict__ track_id, int B, int L, int F, int R,
                                                      const int32_t* __restrict__ off, const int32_t* __restrict__ rank,
                                                      float* __restrict__ rows, int32_t* __restrict__ obj_id) {
    const int b = blockIdx.x;
    const int n = min(max(box_num[b], 0), L);
    const float dx = grm[(size_t)b * 7 + 3], dy = grm[(size_t)b * 7 + 4], dz = grm[(size_t)b * 7 + 5];
    const float label = (float)cls[b];
    const int tid = track_id[b];
    for (int j = threadIdx.x; j < n; j += NT) {
        const size_t e = (size_t)b * L + j;
        const int f = fob[e];
        if (f < 0 || f >= F) continue;
        const int pos = off[(size_t)f * B + b] + rank[e];
        if (pos >= R) continue;
        const double* p = prm + e * 7;
        float* dst = rows + ((size_t)f * R + pos) * 9;
        dst[0] = __double2float_rn(p[0]); dst[1] = __double2float_rn(p[1]); dst[2] = __double2float_rn(p[2]);
        dst[3] = dx; dst[4] = dy; dst[5] = dz;
        dst[6] = __double2float_rn(p[6]);
        dst[7] = score[e];
        dst[8] = label;
        obj_id[(size_t)f * R + pos] = tid;
    }
}

size_t cnt_bytes(int B, int F) { return dz_align_up((size_t)F * B * sizeof(int32_t), 256); }

}  // namespace

extern "C" size_t dz_combine_frames_ws_bytes(int B, int L, int F) {
    return cnt_bytes(B, F) + dz_align_up((size_t)B * L * sizeof(int32_t), 256) + 256;
}

extern "C" int dz_combine_frames(const double* prm_lidar, const float* grm_pred, const float* score, const int32_t* frame_of_box,
                                 const int32_t* box_num, const int32_t* cls, const int32_t* track_id, int B, int L,
                                 const float* det, const int32_t* det_count, const unsigned char* kept, int K, int F, int R,
                                 float* rows, int32_t* obj_id, int32_t* count, int32_t* overflow, void* ws, size_t ws_bytes,
                                 dz_stream_t stream) {
    DZ_CHECK_ARG(B >= 0 && L >= 1 && F >= 1 && R >= 1 && rows && obj_id && count && overflow && ws);
    DZ_CHECK_ARG(B == 0 || (prm_lidar && grm_pred && score && frame_of_box && box_num && cls && track_id));
    DZ_CHECK_ARG(!det || (det_count && kept && K >= 1));
    if (ws_bytes < dz_combine_frames_ws_bytes(B, L, F)) {
        dz_set_error("dz_combine_frames: workspace too small");
        return DZ_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    DzWs w(ws, ws_bytes);
    int32_t* cnt = w.take<int32_t>((size_t)F * B);
    int32_t* rank = w.take<int32_t>((size_t)B * L);
    if (B) DZ_CUDA(cudaMemsetAsync(cnt, 0, (size_t)F * B * sizeof(int32_t), st));
    if (B) {
        k_combine_count<<<B, NT, 0, st>>>(frame_of_box, box_num, B, L, F, cnt, rank, overflow);
        DZ_LAUNCH_CHECK();
    }
    k_combine_frame<<<F, NT, 0, st>>>(cnt, B, det, det_count, kept, K, R, rows, obj_id, count, overflow);
    DZ_LAUNCH_CHECK();
    if (B) {
        k_combine_write<<<B, NT, 0, st>>>(prm_lidar, grm_pred, score, frame_of_box, box_num, cls, track_id, B, L, F, R, cnt, rank, rows,
                                          obj_id);
        DZ_LAUNCH_CHECK();
    }
    return DZ_OK;
}

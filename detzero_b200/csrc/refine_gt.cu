// refine_gt.cu -- the refiners against ground truth on the device (sm_90a): the per-track targets the reference attaches on the
// host, the per-box 3-D IoUs behind the recall records of its three refine models, and the CRM's IoU labels.
//
//   targets   daemon/prepare_object_data.py:64-190 (gt_boxes_global, matched, matched_tracklet, state per track box) and the
//             gt_pos_trajectory of waymo_position_dataset.py:41-42,76-80,159-160.  One thread per box slot.
//   aligned   out[i] = iou3d(a[i], b[i]): what boxes_iou3d_gpu(a, b).diag() keeps of its n x n matrix.
//   score     generate_recall_record of position_refine_model.py:100-133 and geometry_refine_model.py:98-141 (the two
//             boxes_iou3d_gpu(...).diag() calls per track and the per-threshold counts), and generate_refine_boxes_iou of
//             daemon/generate_iou_gt.py:36-53 in label mode.  One block per track, one launch for every track of the call.
//   confidence   the counters of confidence_refine_model.py:81-104.
//
// Deliberate deviation (restated in oracle/refine_score_ref.py): a pair of boxes is re-centred on its ground-truth box centre in
// float64 before it is rounded to float32 for the clip of boxgeom.cuh.  The reference rounds world boxes (GRM, labels) or init-frame
// boxes (PRM) to float32 first; kilometres from the origin a float32 ulp is 5e-4 m, and the IoU does not depend on the frame.
// A ground-truth box without volume scores 0 (the reference's overlap 0 over max(union, 1e-6)).
// The counts are integers, summed by a fixed-order block reduction: bit-identical run to run.
#include "common.cuh"
#include "boxgeom.cuh"
#include "refine_frame.cuh"

namespace {

constexpr int SCORE_NT = 128;
constexpr int MAX_TH = 8;

struct Thresholds { float th[MAX_TH]; int n; };

__device__ __forceinline__ int slots_of(const int* box_num, int b, int L) { return min(max(box_num[b], 0), L); }

}  // namespace

// ---- targets: one thread per box slot ----------------------------------------------------------------------------------------
__global__ void k_refine_targets(const double* __restrict__ gt_world, const int* __restrict__ gt_obj, const int* __restrict__ gt_cnt,
                                 int F, int G, const int* __restrict__ trk_obj, const int* __restrict__ obj_state,
                                 const int* __restrict__ trk_state, const double* __restrict__ boxes, const int* __restrict__ fob,
                                 const int* __restrict__ box_num, int B, int L, double* __restrict__ gt_boxes,
                                 unsigned char* __restrict__ matched, unsigned char* __restrict__ matched_tracklet,
                                 int* __restrict__ state, float* __restrict__ gt_traj) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * L) return;
    const int b = t / L, j = t % L, n = slots_of(box_num, b, L), o = trk_obj[b];
    if (j == 0) {
        matched_tracklet[b] = o >= 0;
        state[b] = o >= 0 ? obj_state[b] : trk_state[b];
    }
    double g[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    unsigned char m = 0;
    if (j < n) {
        if (o < 0) {
            m = 1;                                                        // prepare_object_data.py:184-188
        } else {
            const int f = fob[t];
            if (f >= 0 && f < F) {
                const int ng = min(max(gt_cnt[f], 0), G);
                for (int r = 0; r < ng; ++r) {                            // order_idx[0]: the object's first row of the frame
                    if (gt_obj[(size_t)f * G + r] != o) continue;
                    const double* w = gt_world + ((size_t)f * G + r) * 9;
                    for (int d = 0; d < 7; ++d) g[d] = w[d];
                    m = 1;
                    break;
                }
            }
        }
    }
    matched[t] = m;
    for (int d = 0; d < 7; ++d) gt_boxes[(size_t)t * 7 + d] = g[d];
    float* out = gt_traj + (size_t)t * 7;
    if (j >= n) {
        for (int d = 0; d < 7; ++d) out[d] = 0.f;
        return;
    }
    const double* bi = boxes + ((size_t)b * L + n / 2) * 7;
    double loc[7];
    to_init_frame(init_frame(bi), bi, g, loc);                            // a zero box is transformed too, as the dataset does
    for (int d = 0; d < 7; ++d) out[d] = (float)loc[d];
}

// ---- aligned 3-D IoU -----------------------------------------------------------------------------------------------------------
__global__ void k_iou3d_aligned(const float* __restrict__ A, int lda, const float* __restrict__ Bx, int ldb, int n,
                                float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float a[7], b[7];
#pragma unroll
    for (int d = 0; d < 7; ++d) { a[d] = A[(size_t)i * lda + d]; b[d] = Bx[(size_t)i * ldb + d]; }
    out[i] = iou3d(a, b);
}

// ---- score: one block per track ------------------------------------------------------------------------------------------------
// box (float64 world, dims replaced by `size` when given) against the ground-truth box g, both relative to g's centre
__device__ __forceinline__ float centred_iou(const double* box, const float* size, const double* g) {
    if (!(g[3] * g[4] * g[5] > 0.0)) return 0.f;
    float a[7], c[7];
    for (int d = 0; d < 3; ++d) { a[d] = (float)(box[d] - g[d]); c[d] = 0.f; }
    for (int d = 3; d < 6; ++d) { a[d] = size ? size[d] : (float)box[d]; c[d] = (float)g[d]; }
    a[6] = (float)box[6];
    c[6] = (float)g[6];
    return iou3d(a, c);
}

__global__ void __launch_bounds__(SCORE_NT)
k_refine_score(const double* __restrict__ in_boxes, const double* __restrict__ out_boxes, const float* __restrict__ size,
               const double* __restrict__ gt_boxes, const unsigned char* __restrict__ matched,
               const unsigned char* __restrict__ matched_tracklet, const int* __restrict__ box_num, int L, Thresholds th,
               float* __restrict__ iou_in, float* __restrict__ iou_out, int* __restrict__ rec) {
    const int b = blockIdx.x, n = slots_of(box_num, b, L);
    const bool label = out_boxes == nullptr;
    const bool track_on = label || matched_tracklet[b];
    const float* sz = size ? size + (size_t)b * 7 : nullptr;
    int cnt[1 + 2 * MAX_TH];
#pragma unroll
    for (int k = 0; k < 1 + 2 * MAX_TH; ++k) cnt[k] = 0;
    for (int j = threadIdx.x; j < L; j += SCORE_NT) {
        const size_t t = (size_t)b * L + j;
        float vi = 0.f, vo = 0.f;
        if (j < n && track_on && (label || matched[t])) {
            const double* g = gt_boxes + t * 7;
            vi = centred_iou(in_boxes + t * 7, label ? sz : nullptr, g);
            if (!label) vo = centred_iou(out_boxes + t * 7, sz, g);
            cnt[0] += 1;
#pragma unroll
            for (int k = 0; k < MAX_TH; ++k) {
                if (k < th.n) { cnt[1 + k] += vi > th.th[k]; cnt[1 + MAX_TH + k] += vo > th.th[k]; }
            }
        }
        iou_in[t] = vi;
        if (!label) iou_out[t] = vo;
    }
    if (!rec) return;
    __shared__ int s_cnt[SCORE_NT / 32][1 + 2 * MAX_TH];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 1 + 2 * MAX_TH; ++k) {
        int v = cnt[k];
#pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) s_cnt[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < 1 + 2 * th.n) {
        const int k = threadIdx.x == 0 ? 0 : (threadIdx.x <= th.n ? threadIdx.x : 1 + MAX_TH + (threadIdx.x - 1 - th.n));
        int v = 0;
        for (int w = 0; w < SCORE_NT / 32; ++w) v += s_cnt[w][k];
        rec[(size_t)b * (1 + 2 * th.n) + threadIdx.x] = v;
    }
}

// ---- CRM counters: one warp per track ------------------------------------------------------------------------------------------
__global__ void k_confidence_score(const float* __restrict__ conf, const float* __restrict__ pred, const float* __restrict__ iou,
                                   const int* __restrict__ box_num, int B, int L, int* __restrict__ rec) {
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= B) return;
    const int n = slots_of(box_num, b, L);
    int mu = 0, md = 0, uu = 0;
    for (int j = lane; j < n; j += 32) {
        const size_t t = (size_t)b * L + j;
        const bool lab = iou[t] >= 0.7f, up = pred[t] >= conf[t];
        mu += lab && up;
        md += lab && pred[t] < conf[t];
        uu += iou[t] < 0.7f && up;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        mu += __shfl_xor_sync(0xffffffffu, mu, o);
        md += __shfl_xor_sync(0xffffffffu, md, o);
        uu += __shfl_xor_sync(0xffffffffu, uu, o);
    }
    if (lane == 0) {
        int* r = rec + (size_t)b * 5;
        r[0] = mu; r[1] = md; r[2] = uu; r[3] = n - mu - md - uu; r[4] = n;
    }
}

extern "C" int dz_refine_targets(const double* gt_world, const int32_t* gt_obj, const int32_t* gt_cnt, int F, int G,
                                 const int32_t* trk_obj, const int32_t* obj_state, const int32_t* trk_state, const double* boxes,
                                 const int32_t* frame_of_box, const int32_t* box_num, int B, int L, double* gt_boxes,
                                 unsigned char* matched, unsigned char* matched_tracklet, int32_t* state, float* gt_traj,
                                 dz_stream_t stream) {
    DZ_CHECK_ARG(gt_world && gt_obj && gt_cnt && F >= 1 && G >= 1 && trk_obj && obj_state && trk_state && boxes && frame_of_box &&
                 box_num && B >= 0 && L >= 1 && (long long)B * L < INT_MAX && gt_boxes && matched && matched_tracklet && state &&
                 gt_traj);
    if (B == 0) return DZ_OK;
    k_refine_targets<<<dz_cdiv((long long)B * L, 128), 128, 0, (cudaStream_t)stream>>>(
        gt_world, gt_obj, gt_cnt, F, G, trk_obj, obj_state, trk_state, boxes, frame_of_box, box_num, B, L, gt_boxes, matched,
        matched_tracklet, state, gt_traj);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" int dz_boxes_iou3d_aligned(const float* boxes_a, int lda, const float* boxes_b, int ldb, int n, float* out,
                                      dz_stream_t stream) {
    DZ_CHECK_ARG(boxes_a && boxes_b && out && n >= 0 && lda >= 7 && ldb >= 7);
    if (n == 0) return DZ_OK;
    k_iou3d_aligned<<<dz_cdiv(n, 128), 128, 0, (cudaStream_t)stream>>>(boxes_a, lda, boxes_b, ldb, n, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" int dz_refine_score(const double* in_boxes, const double* out_boxes, const float* size, const double* gt_boxes,
                               const unsigned char* matched, const unsigned char* matched_tracklet, const int32_t* box_num, int B,
                               int L, const double* thresholds, int n_thresholds, float* iou_in, float* iou_out, int32_t* rec,
                               dz_stream_t stream) {
    DZ_CHECK_ARG(in_boxes && gt_boxes && box_num && B >= 0 && L >= 1 && iou_in && n_thresholds >= 0 && n_thresholds <= MAX_TH &&
                 (thresholds || n_thresholds == 0));
    DZ_CHECK_ARG(!out_boxes || (matched && matched_tracklet && iou_out));
    if (B == 0) return DZ_OK;
    Thresholds th;
    th.n = n_thresholds;
    for (int k = 0; k < MAX_TH; ++k) th.th[k] = k < n_thresholds ? (float)thresholds[k] : 0.f;
    k_refine_score<<<B, SCORE_NT, 0, (cudaStream_t)stream>>>(in_boxes, out_boxes, size, gt_boxes, matched, matched_tracklet,
                                                             box_num, L, th, iou_in, iou_out, rec);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" int dz_confidence_score(const float* conf_score, const float* pred_score, const float* iou, const int32_t* box_num,
                                   int B, int L, int32_t* rec, dz_stream_t stream) {
    DZ_CHECK_ARG(conf_score && pred_score && iou && box_num && B >= 0 && L >= 1 && rec);
    if (B == 0) return DZ_OK;
    k_confidence_score<<<dz_cdiv(B, 4), 128, 0, (cudaStream_t)stream>>>(conf_score, pred_score, iou, box_num, B, L, rec);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

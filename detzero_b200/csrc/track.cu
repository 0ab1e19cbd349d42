// track.cu -- the steps either side of the detector / refiner kernels (SURVEY.md §8f rows 2 and 3), sm_90a:
//
//   * tracker association matrices on the device, reading boxes straight from the all-gathered (F, 500, 9) tensor:
//     rotated-BEV IoU, BEV overlap area, 3-D IoU and axis-aligned 2-D IoU.  Replaces
//     tracking/detzero_track/models/tracking_modules/data_association/distance.py:44-141 (IoUBEV_dis_mat / bev_overlap_gpu /
//     IoU3D_dis_mat / IoU2D_dis_mat -> iou3d_nms_cuda.boxes_{iou,overlap}_bev_gpu, iou3d_nms_utils.boxes_iou3d_gpu :74-107),
//     which copy every matrix to the host; the overlap filter of tracking/detzero_track/datasets/data_processor.py:97-163 uses the
//     same overlap matrix.
//   * object crop: which points of a frame fall inside which (enlarged) track box -- points_in_boxes_gpu_v2
//     (utils/detzero_utils/ops/roiaware_pool3d/src/roiaware_pool3d_kernel.cu:23-36,352-372, called from
//     daemon/prepare_object_data.py:264-311) -- plus the ordered compaction the daemon does on the host
//     (`pts[obj_pts_mask[idx]]`): per box the indices of its points in input order, capped, and the true count.  The
//     reference materialises a (T, M) int mask (360 MB for 500 boxes x 180 K points) and copies it to the host.
#include "common.cuh"
#include "boxgeom.cuh"

enum { DZ_PAIR_IOU_BEV = 0, DZ_PAIR_OVERLAP_BEV = 1, DZ_PAIR_IOU_3D = 2, DZ_PAIR_IOU_2D = 3 };

__global__ void k_boxes_pairwise(const float* __restrict__ A, int na, int lda, const float* __restrict__ Bx, int nb, int ldb, int kind,
                                 float* __restrict__ out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= na || j >= nb) return;
    float a[7], b[7];
#pragma unroll
    for (int d = 0; d < 7; ++d) { a[d] = A[(size_t)i * lda + d]; b[d] = Bx[(size_t)j * ldb + d]; }
    float r;
    if (kind == DZ_PAIR_IOU_BEV) {
        r = bev_iou(a, b);                                                       // iou3d_nms_kernel.cu:328-335
    } else if (kind == DZ_PAIR_OVERLAP_BEV) {
        r = bev_overlap(a, b);                                                   // boxes_overlap_bev_gpu
    } else if (kind == DZ_PAIR_IOU_3D) {                                         // iou3d_nms_utils.py:85-105
        r = iou3d(a, b);
    } else {                                                                     // distance.py:69-101 on (x, y, w, h) = box[0,1,3,4]
        const float ax1 = a[0] - a[3] * 0.5f, ay1 = a[1] - a[4] * 0.5f, ax2 = a[0] + a[3] * 0.5f, ay2 = a[1] + a[4] * 0.5f;
        const float bx1 = b[0] - b[3] * 0.5f, by1 = b[1] - b[4] * 0.5f, bx2 = b[0] + b[3] * 0.5f, by2 = b[1] + b[4] * 0.5f;
        const float iw = fmaxf(fminf(ax2, bx2) - fmaxf(ax1, bx1), 0.f), ih = fmaxf(fminf(ay2, by2) - fmaxf(ay1, by1), 0.f);
        const float inter = iw * ih;
        r = inter / (a[3] * a[4] + b[3] * b[4] - inter);
    }
    out[(size_t)i * nb + j] = r;
}

extern "C" int dz_boxes_pairwise(const float* boxes_a, int na, int lda, const float* boxes_b, int nb, int ldb, int kind, float* out,
                                 dz_stream_t stream) {
    DZ_CHECK_ARG(boxes_a && boxes_b && out && na >= 0 && nb >= 0 && lda >= 7 && ldb >= 7 && kind >= 0 && kind <= 3);
    if (na == 0 || nb == 0) return DZ_OK;
    dim3 block(16, 16), grid(dz_cdiv(nb, 16), dz_cdiv(na, 16));
    k_boxes_pairwise<<<grid, block, 0, (cudaStream_t)stream>>>(boxes_a, na, lda, boxes_b, nb, ldb, kind, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---- object crop ----------------------------------------------------------------------------------------------------------
static constexpr int CROP_CHUNK = 2048;            // points per block

// pass 1 (write_idx == 0): counts[t][chunk] = points of the chunk inside box t;  pass 2: ordered indices, starting at the
// exclusive prefix of the box's chunk counts.  Same code for both passes => the same in/out decision for every (box, point).
template <int WRITE>
__global__ void __launch_bounds__(256) k_crop(const float* __restrict__ pts, int n_pts, int pt_stride, const float* __restrict__ boxes, int n_boxes,
                                              int ldb, int* __restrict__ chunk_counts, int n_chunks, int32_t* __restrict__ idx, int cap,
                                              int* __restrict__ num) {
    const int t = blockIdx.y, chunk = blockIdx.x;
    __shared__ float sb[7];
    __shared__ int s_warp[8], s_base;
    if (threadIdx.x < 7) sb[threadIdx.x] = boxes[(size_t)t * ldb + threadIdx.x];
    if (WRITE && threadIdx.x == 0) s_base = chunk_counts[(size_t)t * n_chunks + chunk];      // exclusive prefix (after the scan)
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int run = 0;
    for (int p0 = chunk * CROP_CHUNK; p0 < min(n_pts, (chunk + 1) * CROP_CHUNK); p0 += 256) {
        const int p = p0 + threadIdx.x;
        bool in = false;
        if (p < n_pts) {
            const float* q = pts + (size_t)p * pt_stride;
            in = pt_in_box3d(q[0], q[1], q[2], sb);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, in);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) { const int c = s_warp[w]; before += w < warp ? c : 0; total += c; }
        if (WRITE && in) {
            const int pos = s_base + run + before + __popc(bal & ((1u << lane) - 1u));
            if (pos < cap) idx[(size_t)t * cap + pos] = p;
        }
        run += total;
        __syncthreads();
    }
    if (!WRITE && threadIdx.x == 0) chunk_counts[(size_t)t * n_chunks + chunk] = run;
}

// exclusive scan of every box's chunk counts (in place) + the box's total
__global__ void k_crop_scan(int* __restrict__ chunk_counts, int n_chunks, int* __restrict__ num, int32_t* __restrict__ idx, int cap) {
    const int t = blockIdx.x;
    int* c = chunk_counts + (size_t)t * n_chunks;
    __shared__ int s_tot;
    if (threadIdx.x == 0) {
        int run = 0;
        for (int k = 0; k < n_chunks; ++k) { const int v = c[k]; c[k] = run; run += v; }
        num[t] = run;
        s_tot = run;
    }
    __syncthreads();
    for (int k = min(s_tot, cap) + threadIdx.x; k < cap; k += blockDim.x) idx[(size_t)t * cap + k] = -1;      // padding
}

static int crop_chunks(int n_pts) { return dz_cdiv(max(n_pts, 1), CROP_CHUNK); }

// the per-(box, chunk) counts, scanned in place
static int* carve_crop(DzCarve& cv, int n_pts, int n_boxes) { return cv.take<int>((size_t)n_boxes * crop_chunks(n_pts)); }

extern "C" size_t dz_crop_points_ws_bytes(int n_pts, int n_boxes) { return dz_carve_bytes(carve_crop, n_pts, n_boxes); }

extern "C" int dz_crop_points_in_boxes(const float* points, int n_pts, int pt_stride, const float* boxes, int n_boxes, int ldb,
                                       int32_t* idx, int cap, int* num, void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(points && boxes && idx && num && n_pts >= 0 && n_boxes >= 0 && pt_stride >= 3 && ldb >= 7 && cap >= 1);
    if (n_boxes == 0) return DZ_OK;
    DZ_CHECK_WS(dz_crop_points_ws_bytes(n_pts, n_boxes));
    const int n_chunks = crop_chunks(n_pts);
    DzCarve cv((char*)ws);
    int* cc = carve_crop(cv, n_pts, n_boxes);
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid(n_chunks, n_boxes);
    k_crop<0><<<grid, 256, 0, st>>>(points, n_pts, pt_stride, boxes, n_boxes, ldb, cc, n_chunks, idx, cap, num);
    k_crop_scan<<<n_boxes, 128, 0, st>>>(cc, n_chunks, num, idx, cap);
    k_crop<1><<<grid, 256, 0, st>>>(points, n_pts, pt_stride, boxes, n_boxes, ldb, cc, n_chunks, idx, cap, num);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// the reference's own output form: mask (T, M) int32, 1 where point m is inside box t (points_in_boxes_gpu_v2)
__global__ void __launch_bounds__(256) k_points_in_boxes_mask(const float* __restrict__ pts, int n_pts, int pt_stride, const float* __restrict__ boxes,
                                                              int n_boxes, int ldb, int32_t* __restrict__ mask) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pts) return;
    const float* q = pts + (size_t)p * pt_stride;
    const float x = q[0], y = q[1], z = q[2];
    for (int t = 0; t < n_boxes; ++t) {
        float b[7];
#pragma unroll
        for (int d = 0; d < 7; ++d) b[d] = __ldg(boxes + (size_t)t * ldb + d);
        mask[(size_t)t * n_pts + p] = pt_in_box3d(x, y, z, b) ? 1 : 0;
    }
}

extern "C" int dz_points_in_boxes_mask(const float* points, int n_pts, int pt_stride, const float* boxes, int n_boxes, int ldb,
                                       int32_t* mask, dz_stream_t stream) {
    DZ_CHECK_ARG(points && boxes && mask && n_pts >= 0 && n_boxes >= 0 && pt_stride >= 3 && ldb >= 7);
    if (n_pts == 0 || n_boxes == 0) return DZ_OK;
    k_points_in_boxes_mask<<<dz_cdiv(n_pts, 256), 256, 0, (cudaStream_t)stream>>>(points, n_pts, pt_stride, boxes, n_boxes, ldb, mask);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

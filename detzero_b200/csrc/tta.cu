// tta.cu -- test-time augmentation of the CenterPoint detector on the device (sm_90a):
//
//   * view expansion: B collated frames -> B*V augmented frames (frame b, view v at batch index b*V+v), the augmentations of
//     detection/detzero_det/datasets/augmentor/test_time_augmentor.py:32-100 with the rounding of the reference's float32
//     torch CPU code (rotate_points_along_z, utils/detzero_utils/common_utils.py:220-244: x' = x*c - y*s is evaluated as
//     fma(y, -s, round(x*c)));
//   * box un-augmentation: each view's detections back to the original frame (CenterPoint.test_time_augment,
//     detection/detzero_det/models/centerpoint.py:157-202);
//   * 3-D weighted box fusion of the V views of each frame (weighted_boxes_fusion_3d, detection/detzero_det/utils/
//     ensemble_utils/wbf_3d.py:10-190, called through ensemble.py:7-32 wbf_online).  The reference copies the cluster list to
//     the device and reads one IoU back per input box; here one warp per (frame, label) runs the same sequential clustering
//     with the cluster centres in shared memory.
//
// Every entry point only enqueues work; the explicit __fmul_rn / __fmaf_rn / __fadd_rn / __fdiv_rn keep nvcc from contracting
// the float32 steps whose rounding is pinned.
#include "common.cuh"
#include "boxgeom.cuh"

namespace {

struct TtaViews { float4 p[DZ_TTA_MAX_VIEWS]; };        // x: op (DZ_TTA_*), y, z, w: parameters (see detzero_b200.h)

constexpr float PI_F = 3.14159265358979323846f;
constexpr int WBF_MAX_KEYS = 16384;                      // views * rows per frame: 12 B per key in shared memory
constexpr float WBF_CIRCLE_MARGIN = 0.1f;                // > the 1e-2 in-box margin of the polygon clip (boxgeom.cuh)

int load_views(const float* h_views, int V, TtaViews& tv) {
    for (int v = 0; v < V; ++v) {
        const float* q = h_views + 4 * v;
        const int op = (int)q[0];
        if (op < DZ_TTA_ORIGINAL || op > DZ_TTA_SCALE || q[0] != (float)op) return DZ_ERR_ARG;
        tv.p[v] = make_float4(q[0], q[1], q[2], q[3]);
    }
    return DZ_OK;
}

__global__ void k_tta_expand(const float* __restrict__ in, int n, int stride, int V, TtaViews views, int b, long long out_row0,
                             float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, v = blockIdx.y;
    if (i >= n) return;
    const float* src = in + (size_t)i * stride;
    float* dst = out + ((size_t)out_row0 + (size_t)v * n + i) * stride;
    const float4 q = views.p[v];
    const int op = (int)q.x;
    float x = src[1], y = src[2], z = src[3];
    if (op == DZ_TTA_FLIP_X) {
        y = -y;
    } else if (op == DZ_TTA_FLIP_Y) {
        x = -x;
    } else if (op == DZ_TTA_FLIP_XY) {
        x = -x; y = -y;
    } else if (op == DZ_TTA_ROT) {                       // [x y z] @ [[c s 0] [-s c 0] [0 0 1]]
        const float c = q.y, s = q.z;
        const float xr = __fmaf_rn(y, -s, __fmul_rn(x, c)), yr = __fmaf_rn(y, c, __fmul_rn(x, s));
        x = xr; y = yr;
    } else if (op == DZ_TTA_SCALE) {
        x = __fmul_rn(x, q.y); y = __fmul_rn(y, q.y); z = __fmul_rn(z, q.y);
    }
    dst[0] = (float)(b * V + v);
    dst[1] = x; dst[2] = y; dst[3] = z;
    for (int c = 4; c < stride; ++c) dst[c] = src[c];
}

__global__ void k_tta_unaugment(const float* __restrict__ in, const int* __restrict__ counts, int BV, int K, int V, TtaViews views,
                                float* __restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)BV * K) return;
    const int bv = (int)(idx / K), r = (int)(idx % K);
    float* dst = out + (size_t)idx * 9;
    if (r >= counts[bv]) {
#pragma unroll
        for (int d = 0; d < 9; ++d) dst[d] = 0.f;
        return;
    }
    float x[9];
#pragma unroll
    for (int d = 0; d < 9; ++d) x[d] = in[(size_t)idx * 9 + d];
    const float4 q = views.p[bv % V];
    const int op = (int)q.x;
    if (op == DZ_TTA_FLIP_X) {                           // centerpoint.py:168-170
        x[1] = -x[1]; x[6] = -x[6];
    } else if (op == DZ_TTA_FLIP_Y) {                    // :173-175
        x[0] = -x[0]; x[6] = -__fadd_rn(x[6], PI_F);
    } else if (op == DZ_TTA_FLIP_XY) {                   // :178-180
        x[0] = -x[0]; x[1] = -x[1]; x[6] = __fadd_rn(x[6], PI_F);
    } else if (op == DZ_TTA_ROT) {                       // :183-189: rotate by -a, heading += -a
        const float c = q.y, s = q.z;
        const float xr = __fmaf_rn(x[1], -s, __fmul_rn(x[0], c)), yr = __fmaf_rn(x[1], c, __fmul_rn(x[0], s));
        x[0] = xr; x[1] = yr; x[6] = __fadd_rn(x[6], q.w);
    } else if (op == DZ_TTA_SCALE) {                     // :198-200
#pragma unroll
        for (int d = 0; d < 6; ++d) x[d] = __fdiv_rn(x[d], q.y);
    }
#pragma unroll
    for (int d = 0; d < 9; ++d) dst[d] = x[d];
}

// ---- weighted box fusion ---------------------------------------------------------------------------------------------------
struct WbfParams { double iou_thr[DZ_WBF_MAX_LABELS], skip_thr[DZ_WBF_MAX_LABELS]; };

struct WbfWs {                                    // per frame F = V*K slots; cluster c of label l lives at slot seg[l] + c
    int* order;                                   // (B, F) filtered rows (v*K + r) sorted by (label, score desc, v*K + r)
    int* seg;                                     // (B, L+1) start of each label in `order`, seg[L] = rows kept
    int* ncl;                                     // (B, L) clusters per label
    float* fused;                                 // (B, F, 8) fused box [x..dz, yaw of the first member], label
    float* acc;                                   // (B, F, 8) float32 running sum of score * box (wbf_3d.py:66-70)
    double* conf;                                 // (B, F) float64 score sum
    int* cnt;                                     // (B, F) members
    int* first;                                   // (B, F) cluster slot -> first member (v*K + r)
    int* slot_of;                                 // (B, F) first member (v*K + r) -> cluster slot
};

static WbfWs carve(void* ws, size_t bytes, int B, int F, int L, bool& ok) {
    DzWs w(ws, bytes);
    WbfWs r;
    const size_t BF = (size_t)B * F;
    r.order = w.take<int>(BF); r.seg = w.take<int>((size_t)B * (L + 1)); r.ncl = w.take<int>((size_t)B * L);
    r.fused = w.take<float>(BF * 8); r.acc = w.take<float>(BF * 8); r.conf = w.take<double>(BF); r.cnt = w.take<int>(BF);
    r.first = w.take<int>(BF); r.slot_of = w.take<int>(BF);
    ok = r.order && r.seg && r.ncl && r.fused && r.acc && r.conf && r.cnt && r.first && r.slot_of;
    return r;
}

__device__ __forceinline__ uint32_t desc_key32(float f) {       // ascending key == descending float
    const uint32_t u = __float_as_uint(f);
    return ~((u & 0x80000000u) ? ~u : (u | 0x80000000u));
}

__device__ __forceinline__ unsigned long long desc_key64(double f) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(f);
    return ~((u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull));
}

// ascending bitonic sort of P (a power of two) (key, val) pairs in shared memory; val breaks key ties
__device__ void bitonic_sort(unsigned long long* key, unsigned* val, int P) {
    for (int size = 2; size <= P; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int t = threadIdx.x; t < P / 2; t += blockDim.x) {
                const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const unsigned long long ka = key[lo], kb = key[hi];
                const unsigned va = val[lo], vb = val[hi];
                const bool gt = ka > kb || (ka == kb && va > vb);
                if (gt == up) { key[lo] = kb; key[hi] = ka; val[lo] = vb; val[hi] = va; }
            }
        }
    __syncthreads();
}

// prefilter_boxes (wbf_3d.py:10-53): drop label 0 and labels past L, keep score >= skip_box_thr[label-1], group by label,
// score descending.  Score ties (numpy's quicksort order is not pinned) are broken by (view, row) ascending.
__global__ void __launch_bounds__(1024) k_wbf_prefilter(const float* __restrict__ boxes, const int* __restrict__ counts, int V, int K,
                                                        int L, const __grid_constant__ WbfParams prm, int P, WbfWs w) {
    extern __shared__ unsigned long long sm_key[];
    unsigned* sm_val = (unsigned*)(sm_key + P);
    __shared__ int nf;
    const int b = blockIdx.x, F = V * K;
    if (threadIdx.x == 0) nf = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < F; i += blockDim.x) {
        const int v = i / K, r = i % K;
        if (r >= counts[b * V + v]) continue;
        const float* row = boxes + ((size_t)(b * V + v) * K + r) * 9;
        const int label = (int)row[8];
        const float s = row[7];
        if (label < 1 || label > L || !((double)s >= prm.skip_thr[label - 1])) continue;
        const int pos = atomicAdd(&nf, 1);
        sm_key[pos] = ((unsigned long long)label << 32) | desc_key32(s);
        sm_val[pos] = (unsigned)i;
    }
    __syncthreads();
    const int n = nf;
    for (int i = n + threadIdx.x; i < P; i += blockDim.x) { sm_key[i] = ~0ull; sm_val[i] = ~0u; }
    bitonic_sort(sm_key, sm_val, P);
    int* seg = w.seg + (size_t)b * (L + 1);
    if (n == 0 && threadIdx.x == 0)
        for (int l = 0; l <= L; ++l) seg[l] = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        w.order[(size_t)b * F + i] = (int)sm_val[i];
        const int lab = (int)(sm_key[i] >> 32), prev = i ? (int)(sm_key[i - 1] >> 32) : 0;
        for (int l = prev + 1; l <= lab; ++l) seg[l - 1] = i;
        if (i == n - 1)
            for (int l = lab + 1; l <= L + 1; ++l) seg[l - 1] = n;
    }
}

// the clustering loop of wbf_3d.py:155-169 for one (frame, label), one warp.  find_matching_box (:96-116) takes the first
// argmax of the 3-D IoU against the current fused boxes and joins if it is > iou_thr.  Clusters whose circumscribed BEV
// circles (plus a margin wider than the polygon clip's in-box tolerance) do not meet have IoU exactly 0 there, so they are
// skipped without the clip.  get_weighted_box (:55-93, conf_type 'avg'): float32 member sums of float64 products, a float64
// score sum, the yaw of the first (highest-scoring) member.
__global__ void k_wbf_cluster(const float* __restrict__ boxes, int V, int K, int L, const __grid_constant__ WbfParams prm, WbfWs w) {
    extern __shared__ float3 sm_circ[];                  // fused centre x, y and circumscribed radius per cluster
    const int lab = blockIdx.x, b = blockIdx.y, lane = threadIdx.x, F = V * K;
    const int* seg = w.seg + (size_t)b * (L + 1);
    const int s0 = seg[lab], s1 = seg[lab + 1];
    const size_t base = (size_t)b * F + s0;              // slot of this label's cluster 0
    const double thr = prm.iou_thr[lab];
    int nc = 0;
    for (int j = s0; j < s1; ++j) {
        const int idx = w.order[(size_t)b * F + j];
        const float* row = boxes + ((size_t)(b * V + idx / K) * K + idx % K) * 9;
        float bx[7];
#pragma unroll
        for (int d = 0; d < 7; ++d) bx[d] = row[d];
        const float s = row[7];
        const float rad = 0.5f * sqrtf(bx[3] * bx[3] + bx[4] * bx[4]);
        float best = -1.f;
        int bi = -1;
        for (int c = lane; c < nc; c += 32) {
            const float3 q = sm_circ[c];
            const float dx = q.x - bx[0], dy = q.y - bx[1], reach = q.z + rad + WBF_CIRCLE_MARGIN;
            if (dx * dx + dy * dy > reach * reach) continue;
            const float iou = iou3d(bx, w.fused + (base + c) * 8);
            if (iou > best) { best = iou; bi = c; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob > best || (ob == best && oi >= 0 && (bi < 0 || oi < bi))) { best = ob; bi = oi; }
        }
        if (lane == 0) {
            if (bi >= 0 && (double)best > thr) {
                float* a = w.acc + (base + bi) * 8;
                float* f = w.fused + (base + bi) * 8;
                const double cf = w.conf[base + bi] + (double)s;
#pragma unroll
                for (int d = 0; d < 6; ++d) {
                    a[d] = (float)((double)a[d] + (double)s * (double)bx[d]);
                    f[d] = (float)((double)a[d] / cf);
                }
                w.conf[base + bi] = cf;
                w.cnt[base + bi] += 1;
                sm_circ[bi] = make_float3(f[0], f[1], 0.5f * sqrtf(f[3] * f[3] + f[4] * f[4]));
            } else {
                float* a = w.acc + (base + nc) * 8;
                float* f = w.fused + (base + nc) * 8;
#pragma unroll
                for (int d = 0; d < 7; ++d) { f[d] = bx[d]; a[d] = (float)((double)s * (double)bx[d]); }
                f[7] = (float)(lab + 1);
                w.conf[base + nc] = (double)s;
                w.cnt[base + nc] = 1;
                w.first[base + nc] = idx;
                w.slot_of[(size_t)b * F + idx] = s0 + nc;
                sm_circ[nc] = make_float3(bx[0], bx[1], rad);
            }
        }
        nc += (bi >= 0 && (double)best > thr) ? 0 : 1;
        __syncwarp();
    }
    if (lane == 0) w.ncl[(size_t)b * L + lab] = nc;
}

// wbf_3d.py:171-189: score * min(V, n) / V (allows_overflow=False, unit weights), then all labels by score descending.  The
// float64/float32 steps follow numpy: a single-member cluster keeps its float64 row; a fused row is float32.
__device__ __forceinline__ double wbf_score(double conf, int n, int V) {
    if (n == 1) return conf / (double)V;
    const float w1 = (float)(conf / (double)n);
    const double r = n < V ? (double)__fmul_rn(w1, (float)n) / (double)V : ((double)w1 * (double)V) / (double)V;
    return (double)(float)r;
}

__global__ void __launch_bounds__(1024) k_wbf_output(int V, int K, int L, int P, WbfWs w, float* __restrict__ out,
                                                     int* __restrict__ out_count) {
    extern __shared__ unsigned long long sm_key[];
    unsigned* sm_val = (unsigned*)(sm_key + P);
    const int b = blockIdx.x, F = V * K;
    const int* seg = w.seg + (size_t)b * (L + 1);
    const int* ncl = w.ncl + (size_t)b * L;
    int T = 0;
    for (int l = 0; l < L; ++l) {                        // val = the cluster's first member (v*K + r): unique, breaks score ties
        const int nc = ncl[l];
        for (int c = threadIdx.x; c < nc; c += blockDim.x) {
            const size_t slot = (size_t)b * F + seg[l] + c;
            sm_key[T + c] = desc_key64(wbf_score(w.conf[slot], w.cnt[slot], V));
            sm_val[T + c] = (unsigned)w.first[slot];
        }
        T += nc;
    }
    for (int i = T + threadIdx.x; i < P; i += blockDim.x) { sm_key[i] = ~0ull; sm_val[i] = ~0u; }
    bitonic_sort(sm_key, sm_val, P);
    float* o = out + (size_t)b * F * 9;
    for (int i = threadIdx.x; i < F; i += blockDim.x) {
        float* dst = o + (size_t)i * 9;
        if (i >= T) {
#pragma unroll
            for (int d = 0; d < 9; ++d) dst[d] = 0.f;
            continue;
        }
        const size_t slot = (size_t)b * F + w.slot_of[(size_t)b * F + sm_val[i]];
        const float* f = w.fused + slot * 8;
#pragma unroll
        for (int d = 0; d < 7; ++d) dst[d] = f[d];
        dst[7] = (float)wbf_score(w.conf[slot], w.cnt[slot], V);
        dst[8] = f[7];
    }
    if (threadIdx.x == 0) out_count[b] = T;
}

}  // namespace

extern "C" int dz_tta_expand(const float* points, int stride, const int* h_frame_sizes, int B, const float* h_views, int V, float* out,
                             dz_stream_t stream) {
    DZ_CHECK_ARG(points && out && h_frame_sizes && h_views && stride >= 4 && B >= 1 && V >= 1 && V <= DZ_TTA_MAX_VIEWS);
    TtaViews tv;
    DZ_CHECK_ARG(load_views(h_views, V, tv) == DZ_OK);
    long long start = 0;
    for (int b = 0; b < B; ++b) {
        const int n = h_frame_sizes[b];
        DZ_CHECK_ARG(n >= 0);
        if (n > 0) {
            dim3 grid(dz_cdiv(n, 256), V);
            k_tta_expand<<<grid, 256, 0, (cudaStream_t)stream>>>(points + start * stride, n, stride, V, tv, b, start * V, out);
            DZ_LAUNCH_CHECK();
        }
        start += n;
    }
    return DZ_OK;
}

extern "C" int dz_tta_unaugment(const float* boxes, const int* counts, int BV, int K, const float* h_views, int V, float* out,
                                dz_stream_t stream) {
    DZ_CHECK_ARG(boxes && counts && out && h_views && K >= 1 && V >= 1 && V <= DZ_TTA_MAX_VIEWS && BV >= 0 && BV % V == 0);
    TtaViews tv;
    DZ_CHECK_ARG(load_views(h_views, V, tv) == DZ_OK);
    if (BV == 0) return DZ_OK;
    const long long n = (long long)BV * K;
    k_tta_unaugment<<<dz_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(boxes, counts, BV, K, V, tv, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

static int wbf_pow2(int F) {
    int P = 1;
    while (P < F) P <<= 1;
    return P;
}

extern "C" size_t dz_wbf_3d_ws_bytes(int B, int V, int K, int L) {
    const size_t BF = (size_t)B * V * K;
    return 9 * 256 + BF * (4 + 32 + 32 + 8 + 4 + 4 + 4) + (size_t)B * (2 * L + 1) * 4;
}

extern "C" int dz_wbf_3d(const float* boxes, const int* counts, int B, int V, int K, const double* h_iou_thr, const double* h_skip_thr,
                         int L, float* out, int* out_count, void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(boxes && counts && out && out_count && h_iou_thr && h_skip_thr && B >= 0 && V >= 1 && K >= 1);
    DZ_CHECK_ARG(L >= 1 && L <= DZ_WBF_MAX_LABELS);
    const int F = V * K;
    if ((long long)V * K > WBF_MAX_KEYS) {
        dz_set_error("dz_wbf_3d: views * rows = %lld exceeds %d per frame", (long long)V * K, WBF_MAX_KEYS);
        return DZ_ERR_UNSUPPORTED;
    }
    WbfParams prm;
    for (int l = 0; l < L; ++l) {
        DZ_CHECK_ARG(h_iou_thr[l] >= 0.0);               // the circle test treats a non-meeting cluster as IoU 0 <= thr
        prm.iou_thr[l] = h_iou_thr[l];
        prm.skip_thr[l] = h_skip_thr[l];
    }
    if (B == 0) return DZ_OK;
    bool ok;
    WbfWs w = carve(ws, ws_bytes, B, F, L, ok);
    if (!ok) { dz_set_error("dz_wbf_3d: workspace too small"); return DZ_ERR_WORKSPACE; }
    const int P = wbf_pow2(F);
    const size_t sort_smem = (size_t)P * 12, circ_smem = (size_t)F * sizeof(float3);
    static bool configured = false;
    if (!configured) {
        DZ_CUDA(cudaFuncSetAttribute(k_wbf_prefilter, cudaFuncAttributeMaxDynamicSharedMemorySize, WBF_MAX_KEYS * 12));
        DZ_CUDA(cudaFuncSetAttribute(k_wbf_output, cudaFuncAttributeMaxDynamicSharedMemorySize, WBF_MAX_KEYS * 12));
        DZ_CUDA(cudaFuncSetAttribute(k_wbf_cluster, cudaFuncAttributeMaxDynamicSharedMemorySize, WBF_MAX_KEYS * (int)sizeof(float3)));
        configured = true;
    }
    cudaStream_t st = (cudaStream_t)stream;
    k_wbf_prefilter<<<B, 1024, sort_smem, st>>>(boxes, counts, V, K, L, prm, P, w);
    DZ_LAUNCH_CHECK();
    k_wbf_cluster<<<dim3(L, B), 32, circ_smem, st>>>(boxes, V, K, L, prm, w);
    DZ_LAUNCH_CHECK();
    k_wbf_output<<<B, 1024, sort_smem, st>>>(V, K, L, P, w, out, out_count);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// head.cu -- CenterHead heat-map decode (top-K + box decode) and device-resident rotated-BEV NMS, sm_90a.
//
// Replaces centernet_utils._topk / decode_bbox_from_heatmap (detection/detzero_det/utils/centernet_utils.py:138-230),
// CenterHead.generate_predicted_boxes (center_head.py:315-368), model_nms_utils.class_agnostic_nms
// (model_nms_utils.py:6-25) and iou3d_nms nms_gpu (iou3d_nms_utils.py:154-170, iou3d_nms.cpp:114-160,
// iou3d_nms_kernel.cu:111-232,328-335,386-430).
//
// Design: the reference does 2 x torch.topk + ~20 small kernels + a per-sample Python loop, then NMS with a
// cudaMalloc, a blocking D2H of the suppression mask and a serial CPU scan.  Here: one CTA per (frame, class)
// does a 4-pass radix select + bitonic sort in shared memory, one CTA per frame merges classes, decodes and masks;
// NMS keeps the whole mask in shared memory and runs the serial keep scan on the device.  Nothing syncs the host.
#include "common.cuh"

static constexpr int HD_THREADS = 1024;

__device__ __forceinline__ float sigmoidf_exact(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

// bitonic sort (descending) of n (power of two) 64-bit keys in shared memory
__device__ void bitonic_desc(unsigned long long* keys, int n) {
    for (int k = 2; k <= n; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                int ixj = i ^ j;
                if (ixj > i) {
                    unsigned long long a = keys[i], b = keys[ixj];
                    bool desc = (i & k) == 0;
                    if (desc ? (a < b) : (a > b)) { keys[i] = b; keys[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
}

// per (frame, class): scores -> ws ; top-K by (score desc, index asc) -> cand_keys[(b*C+cls)*Kp + r]
__global__ void __launch_bounds__(HD_THREADS) k_topk_class(const float* __restrict__ head, int HW, int ch, int ch_hm, int ch_iou,
                                                           int use_iou, int num_class, int K, int Kp,
                                                           float* __restrict__ score_ws,
                                                           unsigned long long* __restrict__ cand_keys, const int* __restrict__ overflow) {
    if (overflow && !overflow[blockIdx.x]) return;            // the fast path already produced this (frame, class)
    __shared__ unsigned int hist[256];
    __shared__ unsigned long long keys[1024];
    __shared__ unsigned int sh_prefix, sh_need, sh_cnt;
    const int b = blockIdx.x / num_class, cls = blockIdx.x % num_class;
    const float* hp = head + (size_t)b * HW * ch;
    float* sc = score_ws + ((size_t)b * num_class + cls) * HW;
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {
        float s = sigmoidf_exact(__ldg(hp + (size_t)i * ch + ch_hm + cls));
        if (use_iou) {
            float q = fminf(fmaxf(__ldg(hp + (size_t)i * ch + ch_iou), 0.f), 1.f);    // clamp(iou,0,1)
            s = __fmul_rn(s, __fmul_rn(q, q));                                        // scores * pow(iou, 2)
        }
        sc[i] = s;
    }
    __syncthreads();
    const int Keff = min(K, HW);
    // ---- radix select: find T = Keff-th largest bit pattern, G = #(> T)
    unsigned int prefix = 0, need = Keff;     // need: how many still to take among elements matching prefix
    for (int pass = 0; pass < 4; ++pass) {
        int shift = 24 - 8 * pass;
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        unsigned int himask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
        for (int i = threadIdx.x; i < HW; i += blockDim.x) {
            unsigned int u = __float_as_uint(sc[i]);
            if ((u & himask) == prefix) atomicAdd(&hist[(u >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned int acc = 0; int d = 255;
            for (; d > 0; --d) { if (acc + hist[d] >= need) break; acc += hist[d]; }
            sh_prefix = prefix | ((unsigned int)d << shift);
            sh_need = need - acc;
        }
        __syncthreads();
        prefix = sh_prefix; need = sh_need;
        __syncthreads();
    }
    const unsigned int T = prefix;            // need = how many elements == T to take (lowest indices first)
    // ---- collect > T (any order) then == T in index order
    if (threadIdx.x == 0) sh_cnt = 0;
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) keys[i] = 0ull;
    __syncthreads();
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {
        unsigned int u = __float_as_uint(sc[i]);
        if (u > T) {
            unsigned int pos = atomicAdd(&sh_cnt, 1u);
            keys[pos] = ((unsigned long long)u << 32) | (0xffffffffu - (unsigned int)i);
        }
    }
    __syncthreads();
    unsigned int base = sh_cnt, taken = 0;
    for (int start = 0; start < HW && taken < need; start += blockDim.x) {
        int i = start + threadIdx.x;
        int f = (i < HW && __float_as_uint(sc[i]) == T) ? 1 : 0;
        int tot;
        int ex = block_exclusive_scan(f, &tot);
        if (f && taken + ex < need) keys[base + taken + ex] = ((unsigned long long)T << 32) | (0xffffffffu - (unsigned int)i);
        taken += tot;
    }
    __syncthreads();
    bitonic_desc(keys, Kp);
    for (int i = threadIdx.x; i < Kp; i += blockDim.x) cand_keys[(size_t)blockIdx.x * Kp + i] = i < Keff ? keys[i] : 0ull;
}


// ---- fast path: only scores above SCORE_THRESH can survive the final mask (centernet_utils.py:205-206), and they rank above
// everything else, so top-K can be taken among them.  Pass 1 (whole GPU): score every (frame, class, pixel) and append the
// ones above the threshold to a per-(frame, class) candidate list.  Pass 2 (one CTA per list): exact top-K by
// (score desc, index asc) + bitonic sort.  If a list overflows HD_CAND_CAP the slow full-map kernel below takes over.
static constexpr int HD_CAND_CAP = 4096;

__global__ void __launch_bounds__(256) k_score_prefilter(const float* __restrict__ head, int HW, int ch, int ch_hm, int ch_iou, int use_iou,
                                                         int num_class, int B, float thresh, unsigned long long* __restrict__ cand,
                                                         int* __restrict__ cand_cnt) {
    const long long total = (long long)B * HW;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(t / HW), i = (int)(t % HW);
        const float* px = head + (size_t)t * ch;
        float q2 = 1.f;
        if (use_iou) { float q = fminf(fmaxf(__ldg(px + ch_iou), 0.f), 1.f); q2 = __fmul_rn(q, q); }
        for (int cls = 0; cls < num_class; ++cls) {
            float s = sigmoidf_exact(__ldg(px + ch_hm + cls));
            if (use_iou) s = __fmul_rn(s, q2);
            if (s > thresh) {
                int slot = b * num_class + cls;
                int pos = atomicAdd(cand_cnt + slot, 1);
                if (pos < HD_CAND_CAP)
                    cand[(size_t)slot * HD_CAND_CAP + pos] = ((unsigned long long)__float_as_uint(s) << 32) | (0xffffffffu - (unsigned int)i);
            }
        }
    }
}

// one CTA per (frame, class): sort the candidate list (<= HD_CAND_CAP keys) and keep the K best
__global__ void __launch_bounds__(HD_THREADS) k_topk_from_candidates(const unsigned long long* __restrict__ cand, const int* __restrict__ cand_cnt,
                                                                    int K, int Kp, unsigned long long* __restrict__ cand_keys,
                                                                    int* __restrict__ overflow) {
    __shared__ unsigned long long keys[HD_CAND_CAP];
    const int slot = blockIdx.x;
    const int n = cand_cnt[slot];
    if (n > HD_CAND_CAP) { if (threadIdx.x == 0) overflow[slot] = 1; return; }     // slow path will redo this slot
    if (threadIdx.x == 0) overflow[slot] = 0;
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    if (np2 < Kp) np2 = Kp;
    for (int i = threadIdx.x; i < np2; i += blockDim.x) keys[i] = i < n ? cand[(size_t)slot * HD_CAND_CAP + i] : 0ull;
    __syncthreads();
    bitonic_desc(keys, np2);
    for (int i = threadIdx.x; i < Kp; i += blockDim.x) cand_keys[(size_t)slot * Kp + i] = (i < K && i < n) ? keys[i] : 0ull;
}

struct DecodeGeom {
    float lo[3], vs[3];
    float limit[6];
    float stride;
    float thresh;
};

// per frame: merge the per-class lists, take global top-K, decode, mask, compact (order preserved)
__global__ void __launch_bounds__(HD_THREADS) k_topk_merge_decode(const float* __restrict__ head, int H, int W, int ch, int ch_center,
                                                                  int ch_z, int ch_dim, int ch_rot, int num_class, int K, int Kp,
                                                                  const unsigned long long* __restrict__ cand_keys, DecodeGeom g,
                                                                  float* __restrict__ cand_boxes, float* __restrict__ cand_scores,
                                                                  int32_t* __restrict__ cand_labels, int* __restrict__ d_cand_n) {
    extern __shared__ unsigned long long mkeys[];        // next_pow2(num_class*K)
    const int b = blockIdx.x;
    const int HW = H * W;
    int total = num_class * K, np2 = 1;
    while (np2 < total) np2 <<= 1;
    for (int t = threadIdx.x; t < np2; t += blockDim.x) {
        unsigned long long key = 0ull;
        if (t < total) {
            int cls = t / K, pos = t % K;
            unsigned long long ck = cand_keys[((size_t)b * num_class + cls) * Kp + pos];
            if (ck) key = (ck & 0xffffffff00000000ull) | (unsigned long long)(0xffffffffu - (unsigned int)t);
        }
        mkeys[t] = key;
    }
    __syncthreads();
    bitonic_desc(mkeys, np2);
    const float* hp = head + (size_t)b * HW * ch;
    int written = 0;
    for (int start = 0; start < K; start += blockDim.x) {
        int r = start + threadIdx.x;
        bool ok = false;
        float box[7], score = 0.f; int label = 0;
        if (r < K && mkeys[r]) {
            unsigned long long mk = mkeys[r];
            int t = (int)(0xffffffffu - (unsigned int)(mk & 0xffffffffu));
            int cls = t / K, pos = t % K;
            unsigned long long ck = cand_keys[((size_t)b * num_class + cls) * Kp + pos];
            int idx = (int)(0xffffffffu - (unsigned int)(ck & 0xffffffffu));
            score = __uint_as_float((unsigned int)(mk >> 32));
            label = cls;
            const float* px = hp + (size_t)idx * ch;
            float xs = (float)(idx % W) + __ldg(px + ch_center);
            float ys = (float)(idx / W) + __ldg(px + ch_center + 1);
            // xs * feature_map_stride * voxel_size + range_lo  (centernet_utils.py:190-191), separate roundings
            box[0] = __fadd_rn(__fmul_rn(__fmul_rn(xs, g.stride), g.vs[0]), g.lo[0]);
            box[1] = __fadd_rn(__fmul_rn(__fmul_rn(ys, g.stride), g.vs[1]), g.lo[1]);
            box[2] = __ldg(px + ch_z);
            box[3] = expf(__ldg(px + ch_dim));
            box[4] = expf(__ldg(px + ch_dim + 1));
            box[5] = expf(__ldg(px + ch_dim + 2));
            box[6] = atan2f(__ldg(px + ch_rot + 1), __ldg(px + ch_rot));          // atan2(sin, cos); rot = [cos, sin]
            ok = box[0] >= g.limit[0] && box[1] >= g.limit[1] && box[2] >= g.limit[2] &&
                 box[0] <= g.limit[3] && box[1] <= g.limit[4] && box[2] <= g.limit[5] && score > g.thresh;
        }
        int tot;
        int ex = block_exclusive_scan(ok ? 1 : 0, &tot);
        if (ok) {
            size_t o = (size_t)b * K + written + ex;
#pragma unroll
            for (int d = 0; d < 7; ++d) cand_boxes[o * 7 + d] = box[d];
            cand_scores[o] = score;
            cand_labels[o] = label;
        }
        written += tot;
    }
    if (threadIdx.x == 0) d_cand_n[b] = written;
}

// Kp: K rounded up to a power of two, the top-K sort's size
struct DecodeWs { float* score; unsigned long long *cand_keys, *cand; int *cand_cnt, *overflow, Kp; };

static DecodeWs carve_decode(DzCarve& cv, int B, int H, int W, int num_class, int K) {
    const size_t BC = (size_t)B * num_class;
    DecodeWs w;
    w.Kp = 1;
    while (w.Kp < K) w.Kp <<= 1;
    w.score = cv.take<float>(BC * H * W);
    w.cand_keys = cv.take<unsigned long long>(BC * w.Kp); w.cand = cv.take<unsigned long long>(BC * HD_CAND_CAP);
    w.cand_cnt = cv.take<int>(BC); w.overflow = cv.take<int>(BC);
    return w;
}

extern "C" size_t dz_centerhead_decode_ws_bytes(int B, int H, int W, int num_class, int K) {
    return dz_carve_bytes(carve_decode, B, H, W, num_class, K);
}

extern "C" int dz_centerhead_decode(const float* head, int B, int H, int W, int ch, int ch_center, int ch_z, int ch_dim,
                                    int ch_rot, int ch_iou, int ch_hm, int num_class, int K, const float* range6,
                                    const float* vsize3, int fmap_stride, const float* post_limit6, float score_thresh,
                                    int use_iou, float* cand_boxes, float* cand_scores, int32_t* cand_labels,
                                    int* d_cand_n, void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(head && cand_boxes && cand_scores && cand_labels && d_cand_n && ws);
    DZ_CHECK_ARG(K >= 1 && K <= 1024 && num_class >= 1 && num_class * K <= 4096);
    DZ_CHECK_WS(dz_centerhead_decode_ws_bytes(B, H, W, num_class, K));
    cudaStream_t st = (cudaStream_t)stream;
    DzCarve cv((char*)ws);
    const DecodeWs w = carve_decode(cv, B, H, W, num_class, K);
    const int Kp = w.Kp;
    if (K <= HD_CAND_CAP && score_thresh >= 0.f) {
        DZ_CUDA(cudaMemsetAsync(w.cand_cnt, 0, (size_t)B * num_class * 4, st));
        int blocks = max(1, min(dz_cdiv((long long)B * H * W, 256), DZ_NUM_SMS * 8));
        k_score_prefilter<<<blocks, 256, 0, st>>>(head, H * W, ch, ch_hm, ch_iou, use_iou, num_class, B, score_thresh, w.cand, w.cand_cnt);
        k_topk_from_candidates<<<B * num_class, HD_THREADS, 0, st>>>(w.cand, w.cand_cnt, K, Kp, w.cand_keys, w.overflow);
        k_topk_class<<<B * num_class, HD_THREADS, 0, st>>>(head, H * W, ch, ch_hm, ch_iou, use_iou, num_class, K, Kp, w.score, w.cand_keys, w.overflow);
    } else {
        k_topk_class<<<B * num_class, HD_THREADS, 0, st>>>(head, H * W, ch, ch_hm, ch_iou, use_iou, num_class, K, Kp, w.score, w.cand_keys, nullptr);
    }
    DecodeGeom g;
    for (int d = 0; d < 3; ++d) { g.lo[d] = range6[d]; g.vs[d] = vsize3[d]; }
    for (int d = 0; d < 6; ++d) g.limit[d] = post_limit6[d];
    g.stride = (float)fmap_stride; g.thresh = score_thresh;
    int np2 = 1; while (np2 < num_class * K) np2 <<= 1;
    k_topk_merge_decode<<<B, HD_THREADS, (size_t)np2 * 8, st>>>(head, H, W, ch, ch_center, ch_z, ch_dim, ch_rot, num_class, K, Kp,
                                                                 w.cand_keys, g, cand_boxes, cand_scores, cand_labels, d_cand_n);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// rotated BEV IoU (same geometry as iou3d_nms_kernel.cu:111-232: edge/edge intersections + corners-inside with the
// 1e-2 margin + angular sort + shoelace), written for registers: no local arrays of structs escape to memory.
// ---------------------------------------------------------------------------------------------------------------
#include "boxgeom.cuh"

__global__ void k_boxes_iou(const float* __restrict__ A, int na, const float* __restrict__ Bx, int nb, float* __restrict__ out) {
    int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= na || j >= nb) return;
    float a[7], b[7];
#pragma unroll
    for (int d = 0; d < 7; ++d) { a[d] = A[(size_t)i * 7 + d]; b[d] = Bx[(size_t)j * 7 + d]; }
    out[(size_t)i * nb + j] = bev_iou(a, b);
}

extern "C" int dz_boxes_iou_bev(const float* boxes_a, int na, const float* boxes_b, int nb, float* out, dz_stream_t stream) {
    DZ_CHECK_ARG(boxes_a && boxes_b && out && na >= 0 && nb >= 0);
    if (na == 0 || nb == 0) return DZ_OK;
    dim3 block(16, 16), grid(dz_cdiv(nb, 16), dz_cdiv(na, 16));
    k_boxes_iou<<<grid, block, 0, (cudaStream_t)stream>>>(boxes_a, na, boxes_b, nb, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// suppression mask: mask[b][i][cb] bit jj set iff j = cb*64+jj > i and IoU(i,j) > thresh.
// One warp per row box, a lane per column box (two columns each): the rotated-IoU polygon clipping is ~2-3 K cycles per
// pair, so the pairs are spread over cap/8 x col_blocks CTAs instead of 64 pairs per thread.
__global__ void __launch_bounds__(256) k_nms_mask(const float* __restrict__ boxes, const int* __restrict__ d_n, int cap, float thresh,
                                                 unsigned long long* __restrict__ mask) {
    const int b = blockIdx.z, cb = blockIdx.x;
    const int n = min(d_n[b], cap);
    const int col_blocks = (cap + 63) / 64;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row0 = blockIdx.y * 8, i = row0 + warp;
    const int rb = row0 >> 6;                        // the CTA's 8 rows lie in one 64-block
    if (cb < rb || row0 >= n) return;                // CTA-uniform
    __shared__ float cbox[64 * 7];
    const float* fb = boxes + (size_t)b * cap * 7;
    const int cols = min(64, n - cb * 64);
    if (cols <= 0) {
        if (i < n && lane == 0) mask[((size_t)b * cap + i) * col_blocks + cb] = 0ull;
        return;
    }
    for (int t = threadIdx.x; t < cols * 7; t += blockDim.x) cbox[t] = fb[(size_t)cb * 64 * 7 + t];
    __syncthreads();
    if (i >= n) return;                              // warp-uniform
    float me[7];
#pragma unroll
    for (int d = 0; d < 7; ++d) me[d] = __ldg(fb + (size_t)i * 7 + d);
    const bool v0 = lane < cols && cb * 64 + lane > i;
    const bool v1 = lane + 32 < cols && cb * 64 + lane + 32 > i;
    const bool h0 = v0 && bev_iou(me, cbox + lane * 7) > thresh;
    const bool h1 = v1 && bev_iou(me, cbox + (lane + 32) * 7) > thresh;
    const unsigned lo = __ballot_sync(0xffffffffu, h0), hi = __ballot_sync(0xffffffffu, h1);
    if (lane == 0) mask[((size_t)b * cap + i) * col_blocks + cb] = (unsigned long long)lo | ((unsigned long long)hi << 32);
}

// serial keep scan on the device + output assembly
__global__ void __launch_bounds__(256) k_nms_scan(const float* __restrict__ boxes, const float* __restrict__ scores,
                                                  const int32_t* __restrict__ labels, const int* __restrict__ d_n, int cap,
                                                  const unsigned long long* __restrict__ mask, int post_max, int label_offset,
                                                  float* __restrict__ out, int* __restrict__ d_out_n) {
    extern __shared__ unsigned long long smask[];     // n * col_blocks, then keep list
    const int b = blockIdx.x;
    const int n = min(d_n[b], cap);
    const int col_blocks = (cap + 63) / 64;
    int* keep = reinterpret_cast<int*>(smask + (size_t)cap * col_blocks);
    __shared__ int n_keep;
    for (int t = threadIdx.x; t < n * col_blocks; t += blockDim.x) {
        int i = t / col_blocks, cb = t % col_blocks;
        smask[t] = (cb >= i / 64) ? mask[((size_t)b * cap + i) * col_blocks + cb] : 0ull;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        // lane l owns removed-word l (col_blocks <= 32).  Per 64-box block: resolve the suppression inside the block on its
        // diagonal word (64 dependent steps on registers + one shared-memory read each), then OR the rows of the boxes that
        // were kept into every lane's word -- instead of one shuffle + dependent read per box over all n boxes.
        unsigned long long remv = 0ull;
        int nk = 0;
        const int lane = threadIdx.x;
        for (int blk = 0; blk * 64 < n; ++blk) {
            unsigned long long word = __shfl_sync(0xffffffffu, remv, blk);      // suppressed so far inside this block
            unsigned long long kept = 0ull;
            const int cnt = min(64, n - blk * 64);
            for (int t = 0; t < cnt; ++t) {
                if (!((word >> t) & 1ull)) {
                    kept |= 1ull << t;
                    word |= smask[(size_t)(blk * 64 + t) * col_blocks + blk];
                }
            }
            // every lane computed the same `kept`; record the kept boxes and fold their rows into the removed words
            unsigned long long kk = kept;
            while (kk) {
                const int t = __ffsll((long long)kk) - 1;
                kk &= kk - 1;
                if (lane == 0) keep[nk] = blk * 64 + t;
                ++nk;
                if (lane < col_blocks && lane > blk) remv |= smask[(size_t)(blk * 64 + t) * col_blocks + lane];
            }
        }
        if (threadIdx.x == 0) n_keep = nk;
    }
    __syncthreads();
    const int nk = min(n_keep, post_max);
    float* ob = out + (size_t)b * post_max * 9;
    for (int t = threadIdx.x; t < post_max * 9; t += blockDim.x) {
        int r = t / 9, d = t % 9;
        float v = 0.f;
        if (r < nk) {
            int i = keep[r];
            size_t src = (size_t)b * cap + i;
            v = d < 7 ? boxes[src * 7 + d] : (d == 7 ? scores[src] : (float)(labels[src] + label_offset));
        }
        ob[t] = v;
    }
    if (threadIdx.x == 0) d_out_n[b] = nk;
}

// the suppression mask (B, cap, col_blocks)
static unsigned long long* carve_nms(DzCarve& cv, int B, int cap) { return cv.take<unsigned long long>((size_t)B * cap * ((cap + 63) / 64)); }

extern "C" size_t dz_nms_bev_ws_bytes(int B, int cap) { return dz_carve_bytes(carve_nms, B, cap); }

extern "C" int dz_nms_bev(const float* boxes, const float* scores, const int32_t* labels, const int* d_n, int B, int cap,
                          float thresh, int post_max, int label_offset, float* out, int* d_out_n, void* ws,
                          size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(boxes && scores && labels && d_n && out && d_out_n && ws && B >= 1 && cap >= 1 && cap <= 2048 && post_max >= 1);
    DZ_CHECK_WS(dz_nms_bev_ws_bytes(B, cap));
    cudaStream_t st = (cudaStream_t)stream;
    int col_blocks = (cap + 63) / 64;
    DzCarve cv((char*)ws);
    unsigned long long* mask = carve_nms(cv, B, cap);
    // refuse an unsupported cap before anything is enqueued: a rejected call leaves the workspace and the outputs as they were
    size_t smem = (size_t)cap * col_blocks * 8 + (size_t)cap * 4;
    if (smem > 200 * 1024) { dz_set_error("dz_nms_bev: cap too large for shared-memory scan"); return DZ_ERR_UNSUPPORTED; }
    static bool configured = false;
    if (!configured) {
        DZ_CUDA(cudaFuncSetAttribute(k_nms_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        configured = true;
    }
    dim3 grid(col_blocks, dz_cdiv(cap, 8), B);
    k_nms_mask<<<grid, 256, 0, st>>>(boxes, d_n, cap, thresh, mask);
    k_nms_scan<<<B, 256, smem, st>>>(boxes, scores, labels, d_n, cap, mask, post_max, label_offset, out, d_out_n);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// det_eval.cu -- Waymo-style detection AP / APH records on the device (sm_90a): the counts behind DetZero's evaluator
// (evaluator/detzero_eval.py -> WaymoDetectionMetricsEstimator, detection/detzero_det/datasets/waymo/waymo_eval_detection.py),
// whose Waymo metric library is not available; the metric is restated here as follows.
//
// Shards: OBJECT_TYPE (bit 0 of breakdown_mask) has one shard per Waymo type 1..4 (vehicle, pedestrian, sign, cyclist); RANGE
// (bit 1) has type x [0, 30) / [30, 50) / [50, +inf) of the box centre's sqrt(x^2 + y^2) (float32, no FMA contraction); shard s of the
// records is type - 1 for OBJECT_TYPE and 4 + 3 (type - 1) + range for RANGE.  Cutoff k (0..100) is float32(k * 0.01), the last 1.0;
// a prediction is active at k when its score >= the cutoff.  Per (frame, shard, cutoff) the shard's ground truth is matched to the
// active predictions of its type (of every range) by the maximum sum of IoU over the pairs with IoU >= the type's threshold (0.7
// vehicle, 0.5 otherwise; iou3d or bev_iou of boxgeom.cuh).  At LEVEL_L a ground truth counts when its level <= L (a level other
// than 2 is 1): TP a matched pair whose ground truth counts (a pair whose ground truth does not count is neither TP nor FP), FN an
// unmatched counting ground truth, FP an active prediction of the shard's type matched to nothing -- for RANGE, matched in none of
// the type's three range matchings, and counted in the shard of its own range.  TPH sums each TP's heading accuracy
// 1 - min(d, 2 pi - d) / pi (d the float64 heading difference folded into [0, 2 pi)) rounded to a 2^-32 fixed point.
//
// Persistent blocks over frames.  Per frame: every same-type (ground truth, prediction) pair that is not a far_pair gets its IoU,
// and the valid ones (>= threshold) go into the block's edge scratch of max_pairs.  Per breakdown: union-find components of the
// valid edges (a range breakdown gives each prediction one node per ground-truth range, so the three range graphs stay apart).  A
// component's matching only changes where the cutoff crosses one of its predictions' scores, so it is solved once per distinct
// active set and applied to that cutoff interval: a single edge in closed form, up to SMALL_EDGES edges by the Hungarian of
// assign.cuh on one thread, larger ones on the whole block (cost -IoU for a valid pair, 0 otherwise, rows the smaller side; a
// chosen pair with cost 0 is not a match).  Matches mark per-node cutoff bitmasks; the unmatched runs of those masks give FN and
// FP, so a prediction without a valid edge is an FP at every cutoff it is active without any matching.  Counts go into block-local
// difference arrays over the cutoffs, which are prefix-summed at the end and added to the int64 records with integer atomics:
// the records are identical run to run and whatever the grouping of frames into calls.
//
// Capacity: past max_pairs valid edges in a frame (bit 1) or the SCR_CAP assignment scratch (bit 2) the kernel sets *overflow and
// the records are invalid.
#include "common.cuh"
#include "boxgeom.cuh"
#include "assign.cuh"
#include "eval_common.cuh"

namespace {

constexpr int NT = 256;
constexpr int MAX_BLOCKS = 2 * DZ_NUM_SMS;
constexpr int NK = 101;                     // score cutoffs
constexpr int NKD = NK + 1;                 // difference slots
constexpr int NSHARD = 16;
constexpr int WORDS = 4;                    // cutoff bitmask words per node
constexpr int SMALL_EDGES = 16;             // components with more edges are solved by the whole block
constexpr int SMALL_CAP = SMALL_EDGES + 2;
// solve_small's scratch: a component has at most SMALL_EDGES + 1 nodes, and no split of them into rows and columns takes more
constexpr int SMALL_SCR = hungarian_scratch(SMALL_CAP / 2, SMALL_CAP / 2 + 1);
constexpr int SCR_CAP = 1 << 16;            // float64 assignment scratch per block
constexpr double TWO_PI = 6.283185307179586;
constexpr double PI = 3.141592653589793;

struct Shared {
    int overflow, n_edges, changed;
    float cut[NK];
    int present[NKD];
    HungShared<NT> hs;
};

struct Ws {
    unsigned long long* diff;   // (16, 2, 4, NKD) [TP, FP, FN, TPH] differences over the cutoffs
    int *eg, *ep, *sg, *sp;     // valid edges, then sorted by component
    float *eiou, *siou;
    int *lab, *rcnt, *rlist, *rmap, *clist, *cmap, *alist, *amap, *pkc, *pbin, *gbin;
    unsigned *gbits, *pbits;    // (G | R, WORDS) matched-at-cutoff masks
    double* scr;
};

struct EvIn {
    const float* pred;          // (NF, R, 9)
    const int* pred_cnt;
    const float* gt_box;        // (NF, G, 7)
    const int *gt_type, *gt_level, *gt_cnt;
    int NF, R, G, bev, mask, P;
};

// one block's workspace; carved from a null base it only sizes it (block_ws_bytes)
__host__ __device__ Ws carve(DzCarve& c, int R, int G, int P) {
    Ws w;
    w.diff = c.take<unsigned long long>((size_t)NSHARD * 2 * 4 * NKD);
    w.eg = c.take<int>((size_t)P * 6); w.ep = w.eg + P; w.sg = w.ep + P; w.sp = w.sg + P;
    w.eiou = (float*)(w.sp + P); w.siou = w.eiou + P;
    w.lab = c.take<int>((size_t)G + 3 * R);
    w.rcnt = c.take<int>((size_t)G * 4); w.rlist = w.rcnt + G; w.rmap = w.rlist + G; w.gbin = w.rmap + G;
    w.clist = c.take<int>((size_t)R * 6); w.cmap = w.clist + R; w.alist = w.cmap + R; w.amap = w.alist + R; w.pkc = w.amap + R;
    w.pbin = w.pkc + R;
    w.gbits = c.take<unsigned>((size_t)G * WORDS); w.pbits = c.take<unsigned>((size_t)R * WORDS);
    w.scr = c.take<double>(SCR_CAP);
    return w;
}

size_t block_ws_bytes(int R, int G, int P) {
    DzCarve c(nullptr);
    carve(c, R, G, P);
    return c.bytes;
}

__device__ __forceinline__ int valid_type(int t) { return t >= 1 && t <= 4; }

// heading accuracy of a TP as a 2^-32 fixed point
__device__ __forceinline__ unsigned long long heading_acc(float hp, float hg) {
    double d = fmod(__dadd_rn((double)hp, -(double)hg), TWO_PI);
    if (d < 0.) d = __dadd_rn(d, TWO_PI);
    const double a = __dadd_rn(1., -__ddiv_rn(fmin(d, __dadd_rn(TWO_PI, -d)), PI));
    return (unsigned long long)__double2ll_rn(__dmul_rn(a, 4294967296.));
}

__device__ __forceinline__ void add_interval(unsigned long long* diff, int shard, int lvl, int field, int lo, int hi,
                                             unsigned long long v) {
    unsigned long long* row = diff + ((size_t)(shard * 2 + lvl) * 4 + field) * NKD;
    atomicAdd(row + lo, v);
    atomicAdd(row + hi, 0ull - v);
}

__device__ __forceinline__ void set_bits(unsigned* w, int lo, int hi) {
    for (int i = lo >> 5; i <= (hi - 1) >> 5; ++i) {
        const int a = max(lo - 32 * i, 0), b = min(hi - 32 * i, 32);
        const unsigned m = (b == 32 ? ~0u : ((1u << b) - 1u)) & ~((1u << a) - 1u);
        atomicOr(&w[i], m);
    }
}

__device__ __forceinline__ bool bit(const unsigned* w, int k) { return (w[k >> 5] >> (k & 31)) & 1u; }

// the unmatched runs [s, e) of a node's mask within [0, n)
template <class Emit>
__device__ void unmatched_runs(const unsigned* w, int n, Emit emit) {
    int k = 0;
    while (k < n) {
        while (k < n && bit(w, k)) ++k;
        const int s = k;
        while (k < n && !bit(w, k)) ++k;
        if (k > s) emit(s, k);
    }
}

__device__ __forceinline__ int gt_lvl(const EvIn& in, size_t r) { return in.gt_level[r] == 2 ? 2 : 1; }

// ground truth g matched to prediction p at the cutoffs [lo, hi) of breakdown bd
__device__ void record_match(const EvIn& in, const Ws& w, int f, int bd, int g, int p, int lo, int hi) {
    const size_t gr = (size_t)f * in.G + g;
    const float* pb = in.pred + ((size_t)f * in.R + p) * 9;
    const int t = in.gt_type[gr], lv = gt_lvl(in, gr);
    const int shard = bd ? 4 + 3 * (t - 1) + w.gbin[g] : t - 1;
    const unsigned long long acc = heading_acc(pb[6], in.gt_box[gr * 7 + 6]);
    for (int l = lv - 1; l < 2; ++l) {
        add_interval(w.diff, shard, l, 0, lo, hi, 1ull);
        add_interval(w.diff, shard, l, 3, lo, hi, acc);
    }
    set_bits(w.gbits + (size_t)g * WORDS, lo, hi);
    set_bits(w.pbits + (size_t)p * WORDS, lo, hi);
}

// one component of m <= SMALL_EDGES edges (sorted by ground truth, then prediction) on one thread
__device__ void solve_small(const EvIn& in, const Ws& w, int f, int bd, const int* er, const int* ec, const float* ea, int m) {
    int rows[SMALL_CAP], cols[SMALL_CAP], ckc[SMALL_CAP], eri[SMALL_EDGES], eci[SMALL_EDGES], th[SMALL_CAP], amap[SMALL_CAP];
    int nr = 0, nc = 0, nth = 0;
    for (int i = 0; i < m; ++i) {
        if (i == 0 || er[i] != er[i - 1]) rows[nr++] = er[i];
        eri[i] = nr - 1;
        int c = 0;
        while (c < nc && cols[c] != ec[i]) ++c;
        if (c == nc) { cols[nc] = ec[i]; ckc[nc] = w.pkc[ec[i]]; ++nc; }
        eci[i] = c;
    }
    for (int c = 0; c < nc; ++c) {                                    // distinct activity counts, descending
        const int v = ckc[c];
        int j = 0;
        while (j < nth && th[j] > v) ++j;
        if (j < nth && th[j] == v) continue;
        for (int q = nth; q > j; --q) th[q] = th[q - 1];
        th[j] = v; ++nth;
    }
    double scr[SMALL_SCR];
    for (int j = 0; j < nth && th[j] > 0; ++j) {
        const int hi = th[j], lo = j + 1 < nth ? th[j + 1] : 0;
        int na = 0;
        for (int c = 0; c < nc; ++c) amap[c] = ckc[c] >= hi ? na++ : -1;
        solve_dense(nr, na, m, [&](int i, int& r, int& a, double& cost) {
            r = eri[i]; a = amap[eci[i]]; cost = -(double)ea[i];
            return a >= 0;
        }, 0., 0., scr, [&](int ri, int ai) {
            int c = 0;
            while (amap[c] != ai) ++c;
            record_match(in, w, f, bd, rows[ri], cols[c], lo, hi);
        });
    }
}

__global__ void __launch_bounds__(NT)
k_det_eval(EvIn in, long long* records, int* overflow, char* ws_base, size_t block_bytes) {
    __shared__ Shared sh;
    const int R = in.R, G = in.G, P = in.P;
    DzCarve wc(ws_base + (size_t)blockIdx.x * block_bytes);
    Ws w = carve(wc, R, G, P);
    for (int i = threadIdx.x; i < NSHARD * 2 * 4 * NKD; i += NT) w.diff[i] = 0ull;
    for (int k = threadIdx.x; k < NK; k += NT) sh.cut[k] = score_cutoff(k);
    if (threadIdx.x == 0) sh.overflow = 0;
    __syncthreads();
    for (int f = blockIdx.x; f < in.NF; f += gridDim.x) {
        const int ng = min(max(in.gt_cnt[f], 0), G), np = min(max(in.pred_cnt[f], 0), R);
        const float* pred = in.pred + (size_t)f * R * 9;
        const float* gbox = in.gt_box + (size_t)f * G * 7;
        const int* gtype = in.gt_type + (size_t)f * G;
        if (threadIdx.x == 0) sh.n_edges = 0;
        for (int q = threadIdx.x; q < np; q += NT) {
            const float* b = pred + (size_t)q * 9;
            int kc = 0;
            while (kc < NK && b[7] >= sh.cut[kc]) ++kc;                   // active at the cutoffs k < kc
            w.pkc[q] = kc;
            w.pbin[q] = range_bin(b[0], b[1]);
        }
        for (int g = threadIdx.x; g < ng; g += NT) w.gbin[g] = range_bin(gbox[(size_t)g * 7], gbox[(size_t)g * 7 + 1]);
        __syncthreads();
        // ------------------------------------------------------------ valid edges
        for (long long q = threadIdx.x; q < (long long)ng * np; q += NT) {
            const int g = (int)(q / np), i = (int)(q - (long long)g * np);
            const int t = gtype[g];
            const float* b = pred + (size_t)i * 9;
            if (!valid_type(t) || (int)b[8] != t) continue;
            const float* a = gbox + (size_t)g * 7;
            if (far_pair(a, b)) continue;
            const float iou = in.bev ? bev_iou(a, b) : iou3d(a, b);
            if (!(iou >= (t == 1 ? 0.7f : 0.5f))) continue;
            const int e = atomicAdd(&sh.n_edges, 1);
            if (e >= P) { atomicOr(&sh.overflow, 1); continue; }
            w.eg[e] = g; w.ep[e] = i; w.eiou[e] = iou;
        }
        __syncthreads();
        const int ne = min(sh.n_edges, P);
        for (int bd = 0; bd < 2; ++bd) {
            if (!((in.mask >> bd) & 1)) continue;
            const int nodes = G + (bd ? 3 * R : R);
            auto pnode = [&](int gb, int p) { return G + (bd ? gb * R : 0) + p; };
            for (int v = threadIdx.x; v < nodes; v += NT) w.lab[v] = v;
            for (int g = threadIdx.x; g < ng; g += NT) {
                w.rcnt[g] = 0;
                for (int k = 0; k < WORDS; ++k) w.gbits[(size_t)g * WORDS + k] = 0u;
            }
            for (int q = threadIdx.x; q < np * WORDS; q += NT) w.pbits[q] = 0u;
            __syncthreads();
            uf_label<NT>(w.lab, ne, [&](int e) { return w.eg[e]; }, [&](int e) { return pnode(w.gbin[w.eg[e]], w.ep[e]); }, sh.changed);
            group_edges<NT>(w.lab, ne, ng, w.rcnt, w.eg, w.ep, w.eiou, w.sg, w.sp, w.siou);
            volatile int* lab = w.lab;
            // small components: one thread each
            for (int root = threadIdx.x; root < ng; root += NT) {
                const int end = w.rcnt[root], beg = root ? w.rcnt[root - 1] : 0, m = end - beg;
                if (m == 0 || m > SMALL_EDGES || uf_find(lab, root) != root) continue;
                int* er = w.sg + beg;
                int* ec = w.sp + beg;
                float* ea = w.siou + beg;
                if (m == 1) {
                    if (w.pkc[ec[0]] > 0) record_match(in, w, f, bd, er[0], ec[0], 0, w.pkc[ec[0]]);
                    continue;
                }
                sort_edges(er, ec, ea, m);
                solve_small(in, w, f, bd, er, ec, ea, m);
            }
            __syncthreads();
            // large components: one at a time, the whole block on each
            for (int root = 0; root < ng; ++root) {
                const int end = w.rcnt[root], beg = root ? w.rcnt[root - 1] : 0;
                if (end - beg <= SMALL_EDGES || uf_find(lab, root) != root) continue;
                const int gb = w.gbin[root];
                const int nr = block_compact(ng, [&](int g) { return uf_find(lab, g) == root; },
                                             [&](int g, int pos) { w.rmap[g] = pos; w.rlist[pos] = g; });
                const int nc = block_compact(np, [&](int p) { return uf_find(lab, pnode(gb, p)) == root; },
                                             [&](int p, int pos) { w.cmap[p] = pos; w.clist[pos] = p; });
                for (int k = threadIdx.x; k < NKD; k += NT) sh.present[k] = 0;
                __syncthreads();
                for (int c = threadIdx.x; c < nc; c += NT) sh.present[w.pkc[w.clist[c]]] = 1;
                __syncthreads();
                for (int hi = NK; hi >= 1; --hi) {
                    if (!sh.present[hi]) continue;
                    int lo = hi - 1;
                    while (lo > 0 && !sh.present[lo]) --lo;
                    const int na = block_compact(nc, [&](int c) { return w.pkc[w.clist[c]] >= hi; },
                                                 [&](int c, int pos) { w.amap[c] = pos; w.alist[pos] = c; });
                    if (hungarian_scratch(nr, na) > (size_t)SCR_CAP) {
                        if (threadIdx.x == 0) sh.overflow |= 2;
                        __syncthreads();
                        continue;
                    }
                    solve_dense_block<NT>(nr, na, end - beg, [&](int i, int& ri, int& ai, double& cost) {
                        const int p = w.sp[beg + i];
                        if (w.pkc[p] < hi) return false;
                        ri = w.rmap[w.sg[beg + i]]; ai = w.amap[w.cmap[p]]; cost = -(double)w.siou[beg + i];
                        return true;
                    }, 0., 0., w.scr, sh.hs, [&](int ri, int ai) {
                        record_match(in, w, f, bd, w.rlist[ri], w.clist[w.alist[ai]], lo, hi);
                    });
                    __syncthreads();
                }
            }
            __syncthreads();
            // ------------------------------------------------------------ FN and FP from the unmatched runs
            for (int g = threadIdx.x; g < ng; g += NT) {
                const size_t gr = (size_t)f * G + g;
                const int t = gtype[g];
                if (!valid_type(t)) continue;
                const int shard = bd ? 4 + 3 * (t - 1) + w.gbin[g] : t - 1, lv = gt_lvl(in, gr);
                unmatched_runs(w.gbits + (size_t)g * WORDS, NK, [&](int s, int e) {
                    for (int l = lv - 1; l < 2; ++l) add_interval(w.diff, shard, l, 2, s, e, 1ull);
                });
            }
            for (int q = threadIdx.x; q < np; q += NT) {
                const int t = (int)pred[(size_t)q * 9 + 8];
                if (!valid_type(t) || w.pkc[q] == 0) continue;
                const int shard = bd ? 4 + 3 * (t - 1) + w.pbin[q] : t - 1;
                unmatched_runs(w.pbits + (size_t)q * WORDS, w.pkc[q], [&](int s, int e) {
                    for (int l = 0; l < 2; ++l) add_interval(w.diff, shard, l, 1, s, e, 1ull);
                });
            }
            __syncthreads();
        }
    }
    __syncthreads();
    // ---------------------------------------------------------------- block records -> global records
    for (int row = threadIdx.x; row < NSHARD * 2 * 4; row += NT) {
        const int field = row & 3, sl = row >> 2;                        // sl = shard * 2 + level
        const unsigned long long* d = w.diff + (size_t)row * NKD;
        unsigned long long run = 0;
        for (int k = 0; k < NK; ++k) {
            run += d[k];
            if (run) atomicAdd((unsigned long long*)&records[((size_t)sl * NK + k) * 4 + field], run);
        }
    }
    if (threadIdx.x == 0 && sh.overflow) atomicOr(overflow, sh.overflow);
}

int eval_blocks(int NF) { return NF < MAX_BLOCKS ? NF : MAX_BLOCKS; }

}  // namespace

extern "C" size_t dz_det_eval_ws_bytes(int NF, int R, int G, int max_pairs) {
    if (NF <= 0 || R < 1 || G < 1 || max_pairs < 1) return 256;
    return (size_t)eval_blocks(NF) * block_ws_bytes(R, G, max_pairs) + 256;
}

extern "C" int dz_det_eval(const float* pred, const int* pred_cnt, const float* gt_box, const int* gt_type, const int* gt_level,
                           const int* gt_cnt, int NF, int R, int G, int box_type, int breakdown_mask, int max_pairs, long long* records,
                           int* overflow, void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(pred && pred_cnt && gt_box && gt_type && gt_level && gt_cnt && records && overflow && ws && NF >= 0 && R >= 1 &&
                 G >= 1 && (box_type == 0 || box_type == 1) && breakdown_mask >= 0 && breakdown_mask <= 3 && max_pairs >= 1 &&
                 max_pairs <= (1 << 26) && (long long)G * R < INT_MAX && G + 3LL * R < INT_MAX);
    if (NF == 0 || breakdown_mask == 0) return DZ_OK;
    if (ws_bytes < dz_det_eval_ws_bytes(NF, R, G, max_pairs)) {
        dz_set_error("dz_det_eval: workspace too small");
        return DZ_ERR_WORKSPACE;
    }
    EvIn in{pred, pred_cnt, gt_box, gt_type, gt_level, gt_cnt, NF, R, G, box_type, breakdown_mask, max_pairs};
    char* base = (char*)dz_align_up((size_t)ws, 256);
    k_det_eval<<<eval_blocks(NF), NT, 0, (cudaStream_t)stream>>>(in, records, overflow, base, block_ws_bytes(R, G, max_pairs));
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// track_eval.cu -- Waymo-style tracking records on the device (sm_90a): the counts behind MOTA, MOTP, MISS, MISMATCH and FP of
// DetZero's evaluator in tracking mode (evaluator/detzero_eval.py --tracking -> WaymoTrackingMetricsEstimator,
// evaluator/waymo_eval_tracking.py), whose Waymo metric library is not available; the metric is restated here as CLEAR-MOT:
//
//   chains      matching runs independently per (sequence, Waymo type 1..4, score cutoff k = 0..100: float32(k * 0.01), the last
//               1.0; a prediction is active at k when its score >= the cutoff) over the sequence's frames in order, carrying state
//               from frame to frame.  Level does not affect matching, so one chain serves both levels and both breakdowns.
//   valid pair  a ground-truth row and an active prediction of the chain's type whose iou3d (boxgeom.cuh) is >= the type's
//               threshold (0.7 vehicle, 0.5 otherwise).
//   per frame   1. retention: a pair (object o, prediction id p) this chain matched in the previous frame is kept when o and p are
//                  both present, p is active and the pair is still valid;
//               2. fresh matching of the remaining ground truth against the remaining active predictions by the maximum IoU sum
//                  over valid pairs (cost -IoU for a valid pair, 0 otherwise; a chosen pair with cost 0 is not a match);
//               3. a match (o, p) is a mismatch when o was matched before in this chain, in any earlier frame, and its last matched
//                  prediction id is not p (a gap in o's appearances does not reset this);
//               4. this frame's matches and each matched o's last id become the state of the next frame.
//   LEVEL_L     a ground-truth row counts when its level <= L (a level other than 2 is 1).  A match whose ground truth counts adds
//               a match and 1 - IoU (float64, rounded to a 2^-32 fixed point per match) to the cost, and a mismatch when it is
//               one; an unmatched counting row is a miss; an active prediction matched to nothing is an FP; a prediction matched
//               to a row that does not count is neither.
//   RANGE       (this project's choice, unlike det_eval's RANGE) splits the counts of the type's single chain: matches, misses,
//               mismatches and cost by the range bin (eval_common.cuh range_bin) of the ground-truth box in that frame, an FP by
//               that of the prediction.
//   records     int64 (16 shards, 2 levels, 101 cutoffs, 5) [matches, misses, FP, mismatches, cost in 2^-32 units], shard type - 1
//               for OBJECT_TYPE and 4 + 3 (type - 1) + range for RANGE, as det_eval.cu.
//
// Layout: one block per (type, sequence), the frames in order; thread k < 101 owns the chain of cutoff k.  Per frame the block
// finds the rows of its type, the valid edges with their IoU (independent of the cutoff and the history), and their union-find
// components; retention and activity only remove nodes, so solving each component's remaining subproblem exactly is exact.  A
// component of at most SMALL_EDGES edges (sorted by ground truth, then prediction, so the result does not depend on the edge order)
// is run by every chain thread on its own: a single edge in closed form, otherwise retention by a scan of the edges for each row's
// previous id and the Hungarian of assign.cuh on the rest.  A larger component is run by the whole block, one cutoff at a time,
// with solve_dense_block of assign.cuh (rows and columns compacted in index order).  The chain state, each object's last matched id and frame per
// cutoff, is in the workspace.  Misses and FP are not tracked per row: the block counts the counting ground truth per (range, level)
// and the active predictions per (range, cutoff), and the records take the matched ones off.  Counts go to shared-memory
// accumulators and then to the int64 records by integer atomics, so the records are identical run to run and whatever the grouping
// of sequences into calls.  A chain thread's one-thread solve keeps its scratch on the stack (SMALL_SCR doubles); ptxas reports 72
// bytes of spill stores around it for sm_90a, off the per-frame edge and IoU passes.
//
// Flags (*overflow): bit 1 a frame has more than max_pairs valid edges of one type, bit 2 a component exceeds the assignment
// scratch (the records are then invalid); bit 4 two rows of one frame share a prediction id or a ground-truth object, bit 8 a
// ground-truth object index outside [0, n_obj).
#include "common.cuh"
#include "boxgeom.cuh"
#include "assign.cuh"
#include "eval_common.cuh"

namespace {

constexpr int NT = 128;
constexpr int NK = 101;                     // score cutoffs = chains per (sequence, type)
constexpr int NKD = NK + 1;
constexpr int SMALL_EDGES = 16;             // components with more edges are run by the whole block
constexpr int SMALL_CAP = SMALL_EDGES + 2;
// chain_small's scratch: a component has at most SMALL_EDGES + 1 nodes, and no split of them into rows and columns takes more
constexpr int SMALL_SCR = hungarian_scratch(SMALL_CAP / 2, SMALL_CAP / 2 + 1);
constexpr int SCR_CAP = 1 << 15;            // float64 assignment scratch per block
constexpr double FIXED = 4294967296.;

struct Shared {
    int overflow, n_edges, changed, kmax;
    unsigned long long mt[NK][3][2], mm[NK][3][2], cost[NK][3][2];   // matches, mismatches, cost per (cutoff, gt range, level)
    unsigned long long pm[NK][3];                                    // matched predictions per (cutoff, prediction range)
    unsigned long long act[3][NKD];                                  // predictions per (range, number of active cutoffs)
    unsigned long long ngt[3][2];                                    // counting ground truth per (range, level)
    HungShared<NT> hs;
};

struct Ws {
    int *eg, *ep, *sg, *sp;     // valid edges, then grouped by component
    float *eiou, *siou;
    int *lab, *rcnt, *comp;
    int *gobj, *gbin, *glv, *rret, *rmatch, *rmap, *rlist;
    int *pkc, *pbin, *pid, *cret, *cmap, *clist;
    int *lid, *lf;              // (O, NK) last matched prediction id and frame per object and cutoff
    double* scr;
};

struct TeIn {
    const float* pred;          // (S, F, R, 9)
    const int *pred_id, *pred_cnt;
    const float* gt_box;        // (S, F, G, 7)
    const int *gt_obj, *gt_type, *gt_level, *gt_cnt;
    const int *num_frames, *n_obj;
    int S, F, R, G, O, P, mask;
};

// one block's workspace; carved from a null base it only sizes it (block_ws_bytes)
__host__ __device__ Ws carve(DzCarve& c, int R, int G, int O, int P) {
    Ws w;
    w.eg = c.take<int>((size_t)P * 6); w.ep = w.eg + P; w.sg = w.ep + P; w.sp = w.sg + P;
    w.eiou = (float*)(w.sp + P); w.siou = w.eiou + P;
    w.lab = c.take<int>((size_t)G + R);
    w.rcnt = c.take<int>((size_t)G * 9); w.comp = w.rcnt + G; w.gobj = w.comp + G; w.gbin = w.gobj + G; w.glv = w.gbin + G;
    w.rret = w.glv + G; w.rmatch = w.rret + G; w.rmap = w.rmatch + G; w.rlist = w.rmap + G;
    w.pkc = c.take<int>((size_t)R * 6); w.pbin = w.pkc + R; w.pid = w.pbin + R; w.cret = w.pid + R; w.cmap = w.cret + R;
    w.clist = w.cmap + R;
    w.lid = c.take<int>((size_t)O * NK * 2); w.lf = w.lid + (size_t)O * NK;
    w.scr = c.take<double>(SCR_CAP);
    return w;
}

size_t block_ws_bytes(int R, int G, int O, int P) {
    DzCarve c(nullptr);
    carve(c, R, G, O, P);
    return c.bytes;
}

// ground-truth row g matched to prediction row p in frame f by the chain of cutoff k: counts, then the chain state of g's object
__device__ void record_match(Shared& sh, const Ws& w, int f, int k, int g, int p, float iou) {
    const size_t so = (size_t)w.gobj[g] * NK + k;
    const int id = w.pid[p];
    const bool mis = w.lf[so] >= 0 && w.lid[so] != id;
    const unsigned long long c = (unsigned long long)__double2ll_rn(__dmul_rn(__dadd_rn(1., -(double)iou), FIXED));
    const int b = w.gbin[g];
    for (int l = w.glv[g] - 1; l < 2; ++l) {
        atomicAdd(&sh.mt[k][b][l], 1ull);
        if (mis) atomicAdd(&sh.mm[k][b][l], 1ull);
        atomicAdd(&sh.cost[k][b][l], c);
    }
    atomicAdd(&sh.pm[k][w.pbin[p]], 1ull);
    w.lid[so] = id;
    w.lf[so] = f;
}

__device__ __forceinline__ bool retained(const Ws& w, int f, int k, int g, int p) {
    const size_t so = (size_t)w.gobj[g] * NK + k;
    return w.lf[so] == f - 1 && w.lid[so] == w.pid[p];
}

// the chain of cutoff k on one component of m <= SMALL_EDGES edges (sorted by ground truth, then prediction), on one thread
__device__ void chain_small(Shared& sh, const Ws& w, int f, int k, const int* er, const int* ec, const float* ea, int m) {
    if (m == 1) {
        if (w.pkc[ec[0]] > k) record_match(sh, w, f, k, er[0], ec[0], ea[0]);
        return;
    }
    int cols[SMALL_CAP], eri[SMALL_EDGES], eci[SMALL_EDGES], rmap[SMALL_CAP], amap[SMALL_CAP];
    int mg[SMALL_CAP], mp[SMALL_CAP];
    float mi[SMALL_CAP];
    unsigned char rr[SMALL_CAP], rc[SMALL_CAP];
    int nr = 0, nc = 0, nm = 0;
    for (int i = 0; i < m; ++i) {
        if (i == 0 || er[i] != er[i - 1]) rr[nr++] = 0;
        eri[i] = nr - 1;
        int c = 0;
        while (c < nc && cols[c] != ec[i]) ++c;
        if (c == nc) { rc[nc] = 0; cols[nc++] = ec[i]; }
        eci[i] = c;
    }
    for (int i = 0; i < m; ++i) {                                         // retention
        if (w.pkc[ec[i]] <= k || !retained(w, f, k, er[i], ec[i])) continue;
        rr[eri[i]] = 1; rc[eci[i]] = 1;
        mg[nm] = er[i]; mp[nm] = ec[i]; mi[nm] = ea[i]; ++nm;
    }
    int hr = 0, na = 0;
    for (int r = 0; r < nr; ++r) rmap[r] = rr[r] ? -1 : hr++;
    for (int c = 0; c < nc; ++c) amap[c] = (!rc[c] && w.pkc[cols[c]] > k) ? na++ : -1;
    if (hr && na) {                                                       // fresh matching of the rest
        double scr[SMALL_SCR];
        int rl[SMALL_CAP], al[SMALL_CAP];
        for (int r = 0; r < nr; ++r) if (rmap[r] >= 0) rl[rmap[r]] = r;
        for (int c = 0; c < nc; ++c) if (amap[c] >= 0) al[amap[c]] = c;
        solve_dense(hr, na, m, [&](int i, int& a, int& b, double& cost) {
            a = rmap[eri[i]]; b = amap[eci[i]]; cost = -(double)ea[i];
            return a >= 0 && b >= 0;
        }, 0., 0., scr, [&](int a, int b) {
            const int r = rl[a], c = al[b];
            int i = 0;
            while (eri[i] != r || eci[i] != c) ++i;
            mg[nm] = er[i]; mp[nm] = ec[i]; mi[nm] = ea[i]; ++nm;
        });
    }
    for (int q = 0; q < nm; ++q) record_match(sh, w, f, k, mg[q], mp[q], mi[q]);
}

__global__ void __launch_bounds__(NT)
k_track_eval(TeIn in, long long* records, int* flags, char* ws_base, size_t block_bytes) {
    __shared__ Shared sh;
    const int t = blockIdx.x + 1, s = blockIdx.y;
    const int R = in.R, G = in.G, P = in.P;
    DzCarve wc(ws_base + ((size_t)s * 4 + blockIdx.x) * block_bytes);
    Ws w = carve(wc, R, G, in.O, P);
    const int Fs = min(max(in.num_frames[s], 0), in.F), no = min(max(in.n_obj[s], 0), in.O);
    for (size_t i = threadIdx.x; i < (size_t)no * NK; i += NT) { w.lid[i] = -1; w.lf[i] = -2; }
    for (int i = threadIdx.x; i < NK * 6; i += NT) {
        (&sh.mt[0][0][0])[i] = 0ull; (&sh.mm[0][0][0])[i] = 0ull; (&sh.cost[0][0][0])[i] = 0ull;
    }
    for (int i = threadIdx.x; i < NK * 3; i += NT) (&sh.pm[0][0])[i] = 0ull;
    for (int i = threadIdx.x; i < 3 * NKD; i += NT) (&sh.act[0][0])[i] = 0ull;
    if (threadIdx.x < 6) (&sh.ngt[0][0])[threadIdx.x] = 0ull;
    if (threadIdx.x == 0) sh.overflow = 0;
    __syncthreads();
    for (int f = 0; f < Fs; ++f) {
        const size_t fr = (size_t)s * in.F + f;
        const int ng = min(max(in.gt_cnt[fr], 0), G), np = min(max(in.pred_cnt[fr], 0), R);
        const float* pred = in.pred + fr * R * 9;
        const int* pid = in.pred_id + fr * R;
        const float* gbox = in.gt_box + fr * G * 7;
        const int* gtype = in.gt_type + fr * G;
        const int* gobj = in.gt_obj + fr * G;
        const int* glevel = in.gt_level + fr * G;
        if (threadIdx.x == 0) sh.n_edges = 0;
        // ------------------------------------------------------------ rows of this type
        for (int q = threadIdx.x; q < np; q += NT) {
            const float* b = pred + (size_t)q * 9;
            int kc = -1;
            if ((int)b[8] == t) {
                kc = 0;
                while (kc < NK && b[7] >= score_cutoff(kc)) ++kc;       // active at the cutoffs k < kc
                w.pbin[q] = range_bin(b[0], b[1]);
                atomicAdd(&sh.act[w.pbin[q]][kc], 1ull);
            }
            w.pkc[q] = kc;
            w.pid[q] = pid[q];
            w.cret[q] = 0;
        }
        for (int g = threadIdx.x; g < ng; g += NT) {
            w.rret[g] = 0; w.rmatch[g] = -1;
            if (gtype[g] != t) continue;
            const int o = gobj[g];
            if (o < 0 || o >= no) { atomicOr(&sh.overflow, 8); w.gobj[g] = -1; continue; }
            w.gobj[g] = o;
            w.gbin[g] = range_bin(gbox[(size_t)g * 7], gbox[(size_t)g * 7 + 1]);
            w.glv[g] = glevel[g] == 2 ? 2 : 1;
            for (int l = w.glv[g] - 1; l < 2; ++l) atomicAdd(&sh.ngt[w.gbin[g]][l], 1ull);
        }
        // duplicate ids: each pair (i < j) of rows of valid types is checked by the block of row i's type
        for (long long q = threadIdx.x; q < (long long)np * np; q += NT) {
            const int i = (int)(q / np), j = (int)(q - (long long)i * np);
            if (j <= i || (int)pred[(size_t)i * 9 + 8] != t) continue;
            const int tj = (int)pred[(size_t)j * 9 + 8];
            if (tj >= 1 && tj <= 4 && pid[i] == pid[j]) atomicOr(&sh.overflow, 4);
        }
        for (long long q = threadIdx.x; q < (long long)ng * ng; q += NT) {
            const int i = (int)(q / ng), j = (int)(q - (long long)i * ng);
            if (j <= i || gtype[i] != t) continue;
            if (gtype[j] >= 1 && gtype[j] <= 4 && gobj[i] == gobj[j]) atomicOr(&sh.overflow, 4);
        }
        __syncthreads();
        // ------------------------------------------------------------ valid edges
        for (long long q = threadIdx.x; q < (long long)ng * np; q += NT) {
            const int g = (int)(q / np), i = (int)(q - (long long)g * np);
            if (gtype[g] != t || w.gobj[g] < 0 || w.pkc[i] < 0) continue;
            const float* a = gbox + (size_t)g * 7;
            const float* b = pred + (size_t)i * 9;
            if (far_pair(a, b)) continue;
            const float iou = iou3d(a, b);
            if (!(iou >= (t == 1 ? 0.7f : 0.5f))) continue;
            const int e = atomicAdd(&sh.n_edges, 1);
            if (e >= P) { atomicOr(&sh.overflow, 1); continue; }
            w.eg[e] = g; w.ep[e] = i; w.eiou[e] = iou;
        }
        for (int v = threadIdx.x; v < ng; v += NT) { w.lab[v] = v; w.rcnt[v] = 0; }
        for (int v = threadIdx.x; v < np; v += NT) w.lab[G + v] = G + v;
        __syncthreads();
        const int ne = min(sh.n_edges, P);
        __syncthreads();
        if (ne == 0) continue;
        uf_label<NT>(w.lab, ne, [&](int e) { return w.eg[e]; }, [&](int e) { return G + w.ep[e]; }, sh.changed);
        group_edges<NT>(w.lab, ne, ng, w.rcnt, w.eg, w.ep, w.eiou, w.sg, w.sp, w.siou);
        volatile int* lab = w.lab;
        const int ncomp = block_compact(ng, [&](int g) { return w.rcnt[g] != (g ? w.rcnt[g - 1] : 0); },
                                        [&](int g, int pos) { w.comp[pos] = g; });
        for (int c = threadIdx.x; c < ncomp; c += NT) {                   // sort the small components by (row, prediction)
            const int root = w.comp[c], end = w.rcnt[root], beg = root ? w.rcnt[root - 1] : 0, m = end - beg;
            if (m <= SMALL_EDGES) sort_edges(w.sg + beg, w.sp + beg, w.siou + beg, m);
        }
        __syncthreads();
        // ------------------------------------------------------------ small components: every chain on its own thread
        if (threadIdx.x < NK) {
            const int k = threadIdx.x;
            for (int c = 0; c < ncomp; ++c) {
                const int root = w.comp[c], end = w.rcnt[root], beg = root ? w.rcnt[root - 1] : 0;
                if (end - beg <= SMALL_EDGES) chain_small(sh, w, f, k, w.sg + beg, w.sp + beg, w.siou + beg, end - beg);
            }
        }
        __syncthreads();
        // ------------------------------------------------------------ large components: the whole block, one chain at a time
        for (int c = 0; c < ncomp; ++c) {
            const int root = w.comp[c], end = w.rcnt[root], beg = root ? w.rcnt[root - 1] : 0;
            if (end - beg <= SMALL_EDGES) continue;
            if (threadIdx.x == 0) sh.kmax = 0;
            __syncthreads();
            for (int e = beg + threadIdx.x; e < end; e += NT) atomicMax(&sh.kmax, w.pkc[w.sp[e]]);
            __syncthreads();
            const int kmax = sh.kmax;
            __syncthreads();
            for (int k = 0; k < kmax; ++k) {
                for (int e = beg + threadIdx.x; e < end; e += NT) {       // retention (reads the state of the previous frame)
                    const int g = w.sg[e], p = w.sp[e];
                    if (w.pkc[p] > k && retained(w, f, k, g, p)) { w.rret[g] = 1; w.cret[p] = 1; w.rmatch[g] = e; }
                }
                __syncthreads();
                const int nr = block_compact(ng, [&](int g) { return !w.rret[g] && uf_find(lab, g) == root; },
                                             [&](int g, int pos) { w.rmap[g] = pos; w.rlist[pos] = g; });
                const int na = block_compact(np, [&](int p) { return w.pkc[p] > k && !w.cret[p] && uf_find(lab, G + p) == root; },
                                             [&](int p, int pos) { w.cmap[p] = pos; w.clist[pos] = p; });
                if (nr && na) {
                    if (hungarian_scratch(nr, na) > (size_t)SCR_CAP) {
                        if (threadIdx.x == 0) sh.overflow |= 2;
                    } else {
                        solve_dense_block<NT>(nr, na, end - beg, [&](int i, int& ri, int& ai, double& cost) {
                            const int g = w.sg[beg + i], p = w.sp[beg + i];
                            if (w.pkc[p] <= k || w.rret[g] || w.cret[p]) return false;
                            ri = w.rmap[g]; ai = w.cmap[p]; cost = -(double)w.siou[beg + i];
                            return true;
                        }, 0., 0., w.scr, sh.hs, [&](int ri, int ai) { w.rmatch[w.rlist[ri]] = -2 - w.clist[ai]; });
                    }
                }
                __syncthreads();
                for (int e = beg + threadIdx.x; e < end; e += NT) {       // every match of this chain: counts and state
                    const int g = w.sg[e], p = w.sp[e], r = w.rmatch[g];
                    if (r == e || r == -2 - p) record_match(sh, w, f, k, g, p, w.siou[e]);
                }
                __syncthreads();
                for (int e = beg + threadIdx.x; e < end; e += NT) { w.rret[w.sg[e]] = 0; w.rmatch[w.sg[e]] = -1; w.cret[w.sp[e]] = 0; }
                __syncthreads();
            }
        }
        __syncthreads();
    }
    __syncthreads();
    // ---------------------------------------------------------------- block counts -> records
    if (threadIdx.x < NK) {
        const int k = threadIdx.x;
        unsigned long long tot[4][2][5] = {};
        for (int b = 0; b < 3; ++b) {
            unsigned long long active = 0;
            for (int j = k + 1; j < NKD; ++j) active += sh.act[b][j];
            const unsigned long long fp = active - sh.pm[k][b];
            for (int l = 0; l < 2; ++l) {
                const unsigned long long v[5] = {sh.mt[k][b][l], sh.ngt[b][l] - sh.mt[k][b][l], fp, sh.mm[k][b][l], sh.cost[k][b][l]};
                for (int x = 0; x < 5; ++x) { tot[b][l][x] = v[x]; tot[3][l][x] += v[x]; }
            }
        }
        for (int q = 0; q < 4; ++q) {
            if (!((in.mask >> (q < 3 ? 1 : 0)) & 1)) continue;
            const int shard = q < 3 ? 4 + 3 * (t - 1) + q : t - 1;
            for (int l = 0; l < 2; ++l)
                for (int x = 0; x < 5; ++x)
                    if (tot[q][l][x]) atomicAdd((unsigned long long*)&records[(((size_t)shard * 2 + l) * NK + k) * 5 + x], tot[q][l][x]);
        }
    }
    if (threadIdx.x == 0 && sh.overflow) atomicOr(flags, sh.overflow);
}

__global__ void k_entry_lidar(const double* ent_box, const int* ent_frame, const double* poses, const int* num_frames, int S, int E,
                              int F, float* out) {
    const long long n = (long long)S * E;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int s = (int)(i / E), f = ent_frame[i];
        float* l = out + i * 7;
        if (f < 0 || f >= min(num_frames[s], F)) {
            for (int c = 0; c < 7; ++c) l[c] = 0.f;
            continue;
        }
        entry_to_lidar(ent_box + i * 9, poses + ((size_t)s * F + f) * 16, l);
    }
}

}  // namespace

extern "C" size_t dz_track_eval_ws_bytes(int S, int R, int G, int max_objects, int max_pairs) {
    if (S <= 0 || R < 1 || G < 1 || max_objects < 1 || max_pairs < 1) return 256;
    return (size_t)S * 4 * block_ws_bytes(R, G, max_objects, max_pairs) + 256;
}

extern "C" int dz_track_eval(const float* pred, const int* pred_id, const int* pred_cnt, const float* gt_box, const int* gt_obj,
                             const int* gt_type, const int* gt_level, const int* gt_cnt, const int* num_frames, const int* n_obj, int S,
                             int F, int R, int G, int max_objects, int breakdown_mask, int max_pairs, long long* records, int* flags,
                             void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(pred && pred_id && pred_cnt && gt_box && gt_obj && gt_type && gt_level && gt_cnt && num_frames && n_obj && records &&
                 flags && ws && S >= 0 && S <= 65535 && F >= 1 && R >= 1 && G >= 1 && max_objects >= 1 && breakdown_mask >= 0 &&
                 breakdown_mask <= 3 && max_pairs >= 1 && max_pairs <= (1 << 26) && G + (long long)R < INT_MAX &&
                 (long long)max_objects * NK < INT_MAX);
    if (S == 0 || breakdown_mask == 0) return DZ_OK;
    if (ws_bytes < dz_track_eval_ws_bytes(S, R, G, max_objects, max_pairs)) {
        dz_set_error("dz_track_eval: workspace too small");
        return DZ_ERR_WORKSPACE;
    }
    TeIn in{pred, pred_id, pred_cnt, gt_box, gt_obj, gt_type, gt_level, gt_cnt, num_frames, n_obj, S, F, R, G, max_objects, max_pairs,
            breakdown_mask};
    char* base = (char*)dz_align_up((size_t)ws, 256);
    k_track_eval<<<dim3(4, S), NT, 0, (cudaStream_t)stream>>>(in, records, flags, base, block_ws_bytes(R, G, max_objects, max_pairs));
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" int dz_track_entry_lidar(const double* ent_box, const int* ent_frame, const double* poses, const int* num_frames, int S,
                                    int E, int F, float* out, dz_stream_t stream) {
    DZ_CHECK_ARG(ent_box && ent_frame && poses && num_frames && out && S >= 0 && E >= 0 && F >= 1);
    const long long n = (long long)S * E;
    if (n == 0) return DZ_OK;
    const int blocks = (int)((n + 255) / 256 < 4LL * DZ_NUM_SMS ? (n + 255) / 256 : 4LL * DZ_NUM_SMS);
    k_entry_lidar<<<blocks, 256, 0, (cudaStream_t)stream>>>(ent_box, ent_frame, poses, num_frames, S, E, F, out);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

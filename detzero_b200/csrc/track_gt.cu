// track_gt.cu -- tracks against ground truth on the device (sm_90a): the trajectory scoring shared by DetZero's training-target
// assignment (tracking/detzero_track/models/tracking_modules/target_assign.py:8-139) and its tracklet recall
// (tracking/detzero_track/utils/track_recall.py:153-262, get_trajectory_similarity of utils/track_calculation.py:84-123).
//
// One persistent block per sequence:
//   entries     every track entry's world box goes back to the lidar frame as tracklets_to_frames / transform_boxes3d(inverse=True)
//               do it (entry_to_lidar of eval_common.cuh).  Entries are grouped by frame.
//   objects     per object (a per-sequence index of the rows whose class is scored): trajectory length, first / last row, whether
//               a box is L2 (difficulty 2, or 0 with num_points_in_gt <= 5), and its row in every frame.
//   frames      in ascending order, every (ground-truth row, track entry) pair of the frame of the same class that is not a far
//               pair (boxgeom.cuh) gets its BEV or 3-D IoU; a pair (object, track) with a positive IoU enters a fixed-capacity
//               hash table, whose float32 sum and count are then updated by the one thread that owns the pair in this frame.
//               Assign mode sums the IoUs >= the row's class threshold and counts them; recall mode sums every IoU and counts those
//               >= the threshold.  The frames are separated by block barriers, so each sum accumulates in the reference's frame
//               order and the results are bit-identical run to run and whatever the batch.
//   assignment  similarity = sum / trajectory length (float32) for the pairs with a positive count, cost (double)(1.f - sim);
//               GNN_assignment of the reference (scipy linear_sum_assignment, 5000 where the cost is >= 1) is solved as in
//               tracker.cu: union-find components of the valid edges and the exact Hungarian per component (assign.cuh), on one
//               thread for a small component and on the whole block for a large one.
//   outputs     per object [matched track, match count, trajectory length, L1/L2 bucket, class of the first row]; per track
//               [matched object, class, entry count, dynamic]; per entry the BEV IoU with the matched object in that frame (0
//               where the object is absent or of another class).  An object's bucket is 2 if it is matched and any of its boxes is
//               L2, else that of its first box (track_recall.py:215-258).  The state is dynamic when the matched object's first
//               and last world x-y centres are more than 1 m apart (target_assign.py:117-123, whose speed test is always false).
//
// Capacity: the pair table holds max_pairs pairs per sequence and the assignment scratch SCR_CAP doubles; past either the kernel
// sets overflow[s] (bit 1: pairs, bit 2: scratch) and the results of that sequence are invalid.
#include "common.cuh"
#include "boxgeom.cuh"
#include "assign.cuh"
#include "eval_common.cuh"

namespace {

constexpr int NT = 512;
constexpr int SCR_CAP = 1 << 19;           // float64 assignment scratch per sequence
constexpr int SMALL_EDGES = 32;            // components with more edges are solved by the whole block
constexpr unsigned long long EMPTY = ~0ull;

struct Shared {
    int overflow, n_pairs, n_edges, changed, scr_used, n_list;
    HungShared<NT> hs;
};

struct Ws {
    float* elid;                     // (E, 7) lidar boxes of the entries
    int *ent_trk, *fcnt, *foff, *flist;
    unsigned long long* keys;        // (H) pair keys (object << 32 | track)
    float* psum;
    int* pcnt;
    int *er, *ec, *es_r, *es_c;      // edges, then sorted by component
    float *esim, *es_sim;
    int *lab, *rcnt, *rmap, *cmap, *rlist, *clist;
    int *olen, *ofirst, *olast, *oany2, *orow, *mr, *mc;
    double* scr;
};

__device__ __forceinline__ unsigned pair_hash(int o, int k) { return (unsigned)o * 0x9E3779B1u ^ (unsigned)k * 0x85EBCA77u; }

// slot of the pair (o, k) in the table of H (a power of two) slots; inserts it when `insert`; -1 if absent / the table is full
__device__ int pair_slot(unsigned long long* keys, int H, int o, int k, bool insert, Shared& sh, int P) {
    const unsigned long long key = ((unsigned long long)(unsigned)o << 32) | (unsigned)k;
    unsigned h = pair_hash(o, k) & (unsigned)(H - 1);
    volatile unsigned long long* vk = keys;
    for (int t = 0; t < H; ++t, h = (h + 1) & (unsigned)(H - 1)) {
        const unsigned long long cur = vk[h];
        if (cur == key) return (int)h;
        if (cur != EMPTY) continue;
        if (!insert) return -1;
        const unsigned long long prev = atomicCAS(&keys[h], EMPTY, key);
        if (prev == EMPTY) {
            if (atomicAdd(&sh.n_pairs, 1) >= P) atomicOr(&sh.overflow, 1);
            return (int)h;
        }
        if (prev == key) return (int)h;
    }
    if (insert) atomicOr(&sh.overflow, 1);
    return -1;
}

struct GtIn {
    const float* box;     // (S, F, G, 7) lidar
    const double* world;  // (S, F, G, 9)
    const int *cls, *obj, *diff, *npts;   // (S, F, G)
    const int* cnt;       // (S, F)
    const int* nf;        // (S)
    const int* n_obj;     // (S)
    int F, G, O;
};

struct TkIn {
    const int* trk;       // (S, T, 6)
    const int* n_tracks;  // (S)
    const double* ent_box;  // (S, E, 9)
    const int* ent_frame;   // (S, E)
    const double* poses;  // (S, F, 4, 4)
    int T, E;
};

struct GtOut {
    int* obj_rec;         // (S, O, 5)
    int* trk_rec;         // (S, T, 4)
    float* ent_iou;       // (S, E)
    int* overflow;        // (S)
};

struct GtPar {
    float thr[4];         // per class 1..3
    int class_mask;       // bit c: class c is scored
    int recall, iou3d, P, H;
};

}  // namespace

// one sequence's workspace; carved from a null base it only sizes it (gt_seq_ws_bytes)
static __host__ __device__ Ws carve_gt(DzCarve& c, int F, int O, int T, int E, int P, int H) {
    Ws w;
    w.elid = c.take<float>((size_t)E * 7); w.ent_trk = c.take<int>(E);
    w.fcnt = c.take<int>((size_t)F + 1); w.foff = c.take<int>((size_t)F + 1); w.flist = c.take<int>(E);
    w.keys = c.take<unsigned long long>(H); w.psum = c.take<float>(H); w.pcnt = c.take<int>(H);
    w.er = c.take<int>((size_t)P * 6); w.ec = w.er + P; w.es_r = w.ec + P; w.es_c = w.es_r + P;
    w.esim = (float*)(w.es_c + P); w.es_sim = w.esim + P;
    w.lab = c.take<int>((size_t)O + T); w.rcnt = c.take<int>(O);
    w.rmap = c.take<int>(O); w.cmap = c.take<int>(T); w.rlist = c.take<int>(O); w.clist = c.take<int>(T);
    w.olen = c.take<int>((size_t)O * 4); w.ofirst = w.olen + O; w.olast = w.ofirst + O; w.oany2 = w.olast + O;
    w.orow = c.take<int>((size_t)O * F); w.mr = c.take<int>(O); w.mc = c.take<int>(T);
    w.scr = c.take<double>(SCR_CAP);
    return w;
}

static size_t gt_seq_ws_bytes(int F, int O, int T, int E, int P, int H) {
    DzCarve c(nullptr);
    carve_gt(c, F, O, T, E, P, H);
    return c.bytes + 256;
}

__global__ void __launch_bounds__(NT, 1)
k_track_gt(GtIn gt, TkIn tk, GtPar pr, GtOut out, char* ws_base, size_t seq_bytes) {
    const int s = blockIdx.x;
    const int F = gt.F, G = gt.G, T = tk.T, E = tk.E, P = pr.P, H = pr.H;
    const int O = gt.O;
    __shared__ Shared sh;
    DzCarve wc(ws_base + (size_t)s * seq_bytes);
    Ws w = carve_gt(wc, F, O, T, E, P, H);
    const int nt = min(max(tk.n_tracks[s], 0), T);
    const int no = min(max(gt.n_obj[s], 0), O);
    const int Fs = min(max(gt.nf[s], 0), F);
    const int* trk = tk.trk + (size_t)s * T * 6;
    const double* ebox = tk.ent_box + (size_t)s * E * 9;
    const int* eframe = tk.ent_frame + (size_t)s * E;
    const double* poses = tk.poses + (size_t)s * F * 16;
    const size_t gbase = (size_t)s * F * G;
    const int n_ent = nt ? min(trk[(size_t)(nt - 1) * 6 + 5] + trk[(size_t)(nt - 1) * 6 + 3], E) : 0;
    if (threadIdx.x == 0) { sh.overflow = 0; sh.n_pairs = 0; sh.n_edges = 0; sh.scr_used = 0; }
    for (int i = threadIdx.x; i < H; i += NT) { w.keys[i] = EMPTY; w.psum[i] = 0.f; w.pcnt[i] = 0; }
    for (int o = threadIdx.x; o < no; o += NT) { w.olen[o] = 0; w.ofirst[o] = INT_MAX; w.olast[o] = -1; w.oany2[o] = 0; w.mr[o] = -1; }
    for (size_t i = threadIdx.x; i < (size_t)no * F; i += NT) w.orow[i] = -1;
    for (int f = threadIdx.x; f <= F; f += NT) w.fcnt[f] = 0;
    for (int k = threadIdx.x; k < nt; k += NT) w.mc[k] = -1;
    __syncthreads();
    // ---------------------------------------------------------------- entries: lidar boxes, frame lists
    for (int e = threadIdx.x; e < n_ent; e += NT) {
        int lo = 0, hi = nt - 1;                                     // the track whose entry range holds e
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (trk[(size_t)mid * 6 + 5] <= e) lo = mid; else hi = mid - 1; }
        w.ent_trk[e] = lo;
        const int f = eframe[e];
        const double* b = ebox + (size_t)e * 9;
        float* l = w.elid + (size_t)e * 7;
        if (f < 0 || f >= Fs) continue;
        entry_to_lidar(b, poses + (size_t)f * 16, l);
        atomicAdd(&w.fcnt[f], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int f = 0; f < Fs; ++f) { const int c = w.fcnt[f]; w.foff[f] = run; w.fcnt[f] = run; run += c; }
        w.foff[Fs] = run;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < n_ent; e += NT) {
        const int f = eframe[e];
        if (f >= 0 && f < Fs) w.flist[atomicAdd(&w.fcnt[f], 1)] = e;
    }
    // ---------------------------------------------------------------- objects
    for (long long p = threadIdx.x; p < (long long)Fs * G; p += NT) {
        const int f = (int)(p / G), g = (int)(p - (long long)f * G);
        if (g >= gt.cnt[(size_t)s * F + f]) continue;
        const size_t r = gbase + (size_t)f * G + g;
        const int c = gt.cls[r], o = gt.obj[r];
        if (c < 1 || c > 3 || !((pr.class_mask >> c) & 1) || o < 0 || o >= no) continue;
        atomicAdd(&w.olen[o], 1);
        atomicMin(&w.ofirst[o], (int)p);
        atomicMax(&w.olast[o], (int)p);
        const int d = gt.diff[r] == 0 ? (gt.npts[r] > 5 ? 1 : 2) : gt.diff[r];
        if (d == 2) atomicOr(&w.oany2[o], 1);
        w.orow[(size_t)o * F + f] = g;
    }
    __syncthreads();
    // ---------------------------------------------------------------- frames in ascending order
    for (int f = 0; f < Fs; ++f) {
        const int ng = min(max(gt.cnt[(size_t)s * F + f], 0), G), eb = w.foff[f], ne = w.foff[f + 1] - eb;
        const long long pairs = (long long)ng * ne;
        for (long long p = threadIdx.x; p < pairs; p += NT) {
            const int g = (int)(p / ne), i = (int)(p - (long long)g * ne);
            const size_t r = gbase + (size_t)f * G + g;
            const int c = gt.cls[r], o = gt.obj[r];
            if (c < 1 || c > 3 || !((pr.class_mask >> c) & 1) || o < 0 || o >= no) continue;
            const int e = w.flist[eb + i], k = w.ent_trk[e];
            if (trk[(size_t)k * 6 + 1] != c) continue;                   // distinguish_class: another class scores 0
            const float* a = gt.box + r * 7;
            const float* b = w.elid + (size_t)e * 7;
            if (far_pair(a, b)) continue;
            const float iou = pr.iou3d ? iou3d(a, b) : bev_iou(a, b);
            if (!(iou > 0.f)) continue;
            const int slot = pair_slot(w.keys, H, o, k, true, sh, P);
            if (slot < 0) continue;
            const bool hit = iou >= pr.thr[c];
            if (pr.recall) { w.psum[slot] += iou; w.pcnt[slot] += hit; }
            else if (hit) { w.psum[slot] += iou; w.pcnt[slot] += 1; }
        }
        __syncthreads();
    }
    // ---------------------------------------------------------------- valid edges: similarity sum / length, count > 0
    for (int i = threadIdx.x; i < H; i += NT) {
        const unsigned long long key = w.keys[i];
        if (key == EMPTY || w.pcnt[i] <= 0) continue;
        const int o = (int)(key >> 32), k = (int)(key & 0xffffffffu);
        const int e = atomicAdd(&sh.n_edges, 1);
        if (e >= P) { atomicOr(&sh.overflow, 1); continue; }
        w.er[e] = o; w.ec[e] = k; w.esim[e] = w.psum[i] / (float)w.olen[o];
    }
    for (int v = threadIdx.x; v < no + nt; v += NT) w.lab[v] = v;
    for (int o = threadIdx.x; o < no; o += NT) w.rcnt[o] = 0;
    __syncthreads();
    const int ne = min(sh.n_edges, P);
    uf_label<NT>(w.lab, ne, [&](int e) { return w.er[e]; }, [&](int e) { return no + w.ec[e]; }, sh.changed);
    group_edges<NT>(w.lab, ne, no, w.rcnt, w.er, w.ec, w.esim, w.es_r, w.es_c, w.es_sim);
    volatile int* lab = w.lab;
    // cost (double)(1.f - sim), 5000 off the valid edges; a chosen pair is a match when its cost is below 1
    // small components: one thread each, edges sorted by (object, track)
    for (int root = threadIdx.x; root < no; root += NT) {
        const int end = w.rcnt[root], beg = root ? w.rcnt[root - 1] : 0;
        if (end == beg || uf_find(lab, root) != root) continue;
        int* er = w.es_r + beg;
        int* ec = w.es_c + beg;
        float* ea = w.es_sim + beg;
        const int m = end - beg;
        if (m == 1) { w.mr[er[0]] = ec[0]; continue; }
        if (m > SMALL_EDGES) continue;
        sort_edges(er, ec, ea, m);
        const int need = 3 * m + 8;
        const int base = atomicAdd(&sh.scr_used, need);
        if (base + need > SCR_CAP) { atomicOr(&sh.overflow, 2); continue; }
        int* cols = (int*)(w.scr + base);                                // distinct tracks, ascending
        int nc = 0;
        for (int i = 0; i < m; ++i) {
            const int c = ec[i];
            int j = nc - 1;
            while (j >= 0 && cols[j] > c) --j;
            if (j >= 0 && cols[j] == c) continue;
            for (int k = nc; k > j + 1; --k) cols[k] = cols[k - 1];
            cols[j + 1] = c; ++nc;
        }
        int* rows = cols + nc;
        int nr = 0;
        for (int i = 0; i < m; ++i) if (i == 0 || er[i] != er[i - 1]) rows[nr++] = er[i];
        const int need2 = (int)hungarian_scratch(nr, nc);
        const int base2 = atomicAdd(&sh.scr_used, need2);
        if (base2 + need2 > SCR_CAP) { atomicOr(&sh.overflow, 2); continue; }
        solve_dense(nr, nc, m, [&](int i, int& ri, int& ci, double& cost) {
            ri = 0; ci = 0;
            while (rows[ri] != er[i]) ++ri;
            while (cols[ci] != ec[i]) ++ci;
            cost = (double)(1.f - ea[i]);
            return true;
        }, 5000., 1., w.scr + base2, [&](int ri, int ci) { w.mr[rows[ri]] = cols[ci]; });
    }
    __syncthreads();
    // large components: one at a time, the whole block on each
    for (int root = 0; root < no; ++root) {
        const int end = w.rcnt[root], beg = root ? w.rcnt[root - 1] : 0;
        if (end - beg <= SMALL_EDGES || uf_find(lab, root) != root) continue;
        const int nr = block_compact(no, [&](int r) { return uf_find(lab, r) == root; },
                                     [&](int r, int pos) { w.rmap[r] = pos; w.rlist[pos] = r; });
        const int nc = block_compact(nt, [&](int c) { return uf_find(lab, no + c) == root; },
                                     [&](int c, int pos) { w.cmap[c] = pos; w.clist[pos] = c; });
        const size_t a0 = (size_t)sh.scr_used;                           // the small components' scratch stays untouched
        if (a0 + hungarian_scratch(nr, nc) > (size_t)SCR_CAP) {
            if (threadIdx.x == 0) atomicOr(&sh.overflow, 2);
            __syncthreads();
            continue;
        }
        solve_dense_block<NT>(nr, nc, end - beg, [&](int i, int& ri, int& ci, double& cost) {
            ri = w.rmap[w.es_r[beg + i]]; ci = w.cmap[w.es_c[beg + i]];
            cost = (double)(1.f - w.es_sim[beg + i]);
            return true;
        }, 5000., 1., w.scr + a0, sh.hs, [&](int ri, int ci) { w.mr[w.rlist[ri]] = w.clist[ci]; });
        __syncthreads();
    }
    __syncthreads();
    // ---------------------------------------------------------------- outputs
    for (int o = threadIdx.x; o < no; o += NT) if (w.mr[o] >= 0) w.mc[w.mr[o]] = o;
    __syncthreads();
    int* orec = out.obj_rec + (size_t)s * O * 5;
    for (int o = threadIdx.x; o < no; o += NT) {
        const int k = w.mr[o], len = w.olen[o];
        int cnt = 0, bucket = 0, cls = 0;
        if (len > 0) {
            const int f1 = w.ofirst[o] / G, g1 = w.ofirst[o] - f1 * G;
            const size_t r1 = gbase + (size_t)f1 * G + g1;
            cls = gt.cls[r1];
            const int d1 = gt.diff[r1] == 0 ? (gt.npts[r1] > 5 ? 1 : 2) : gt.diff[r1];
            bucket = k >= 0 ? (w.oany2[o] ? 2 : 1) : d1;
        }
        if (k >= 0) { const int slot = pair_slot(w.keys, H, o, k, false, sh, P); cnt = slot >= 0 ? w.pcnt[slot] : 0; }
        int* rr = orec + (size_t)o * 5;
        rr[0] = k; rr[1] = cnt; rr[2] = len; rr[3] = bucket; rr[4] = cls;
    }
    int* trec = out.trk_rec + (size_t)s * T * 4;
    for (int k = threadIdx.x; k < nt; k += NT) {
        const int o = w.mc[k];
        int dyn = 0;
        if (o >= 0) {
            const int f1 = w.ofirst[o] / G, g1 = w.ofirst[o] - f1 * G, f2 = w.olast[o] / G, g2 = w.olast[o] - f2 * G;
            const double* a = gt.world + (gbase + (size_t)f1 * G + g1) * 9;
            const double* b = gt.world + (gbase + (size_t)f2 * G + g2) * 9;
            const double dx = __dadd_rn(a[0], -b[0]), dy = __dadd_rn(a[1], -b[1]);
            dyn = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy))) > 1.;
        }
        int* rr = trec + (size_t)k * 4;
        rr[0] = o; rr[1] = trk[(size_t)k * 6 + 1]; rr[2] = trk[(size_t)k * 6 + 3]; rr[3] = dyn;
    }
    float* eiou = out.ent_iou + (size_t)s * E;
    for (int e = threadIdx.x; e < n_ent; e += NT) {
        const int k = w.ent_trk[e], o = w.mc[k], f = eframe[e];
        float v = 0.f;
        if (o >= 0 && f >= 0 && f < Fs) {
            const int g = w.orow[(size_t)o * F + f];
            if (g >= 0) {
                const size_t r = gbase + (size_t)f * G + g;
                const float* a = gt.box + r * 7;
                const float* b = w.elid + (size_t)e * 7;
                if (gt.cls[r] == trk[(size_t)k * 6 + 1] && !far_pair(a, b)) v = bev_iou(a, b);
            }
        }
        eiou[e] = v;
    }
    if (threadIdx.x == 0) out.overflow[s] = sh.overflow;
}

static int table_slots(int P) {
    int H = 1;
    while (H < 2 * P) H <<= 1;
    return H;
}

extern "C" size_t dz_track_gt_ws_bytes(int S, int F, int max_objects, int max_tracks, int max_entries, int max_pairs) {
    return (size_t)S * dz_align_up(gt_seq_ws_bytes(F, max_objects, max_tracks, max_entries, max_pairs, table_slots(max_pairs)), 256)
           + 256;
}

extern "C" int dz_track_gt(const float* gt_box, const double* gt_world, const int* gt_cls, const int* gt_obj, const int* gt_diff,
                           const int* gt_npts, const int* gt_cnt, const int* gt_num_frames, const int* n_obj, int S, int F, int G,
                           int max_objects, const int* trk, const int* n_tracks, const double* ent_box, const int* ent_frame,
                           const double* poses, int max_tracks, int max_entries, const double* thresholds, int class_mask,
                           int recall, int iou_3d, int max_pairs, int* obj_rec, int* trk_rec, float* ent_iou, int* overflow, void* ws,
                           size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(gt_box && gt_world && gt_cls && gt_obj && gt_diff && gt_npts && gt_cnt && gt_num_frames && n_obj && trk && n_tracks &&
                 ent_box && ent_frame && poses && thresholds && obj_rec && trk_rec && ent_iou && overflow && ws && S >= 0 && F >= 1 &&
                 G >= 1 && max_objects >= 1 && max_tracks >= 1 && max_entries >= 1 && max_pairs >= 1 && max_pairs <= (1 << 28) &&
                 (long long)F * G < INT_MAX);
    if (S == 0) return DZ_OK;
    if (ws_bytes < dz_track_gt_ws_bytes(S, F, max_objects, max_tracks, max_entries, max_pairs)) {
        dz_set_error("dz_track_gt: workspace too small");
        return DZ_ERR_WORKSPACE;
    }
    GtPar pr;
    pr.thr[0] = 0.f;
    for (int c = 0; c < 3; ++c) pr.thr[c + 1] = (float)thresholds[c];
    pr.class_mask = class_mask; pr.recall = recall; pr.iou3d = iou_3d; pr.P = max_pairs; pr.H = table_slots(max_pairs);
    GtIn gi{gt_box, gt_world, gt_cls, gt_obj, gt_diff, gt_npts, gt_cnt, gt_num_frames, n_obj, F, G, max_objects};
    TkIn ti{trk, n_tracks, ent_box, ent_frame, poses, max_tracks, max_entries};
    GtOut go{obj_rec, trk_rec, ent_iou, overflow};
    const size_t seq_bytes = dz_align_up(gt_seq_ws_bytes(F, max_objects, max_tracks, max_entries, max_pairs, pr.H), 256);
    char* base = (char*)dz_align_up((size_t)ws, 256);
    k_track_gt<<<S, NT, 0, (cudaStream_t)stream>>>(gi, ti, pr, go, base, seq_bytes);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

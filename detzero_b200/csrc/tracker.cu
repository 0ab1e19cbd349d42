// tracker.cu -- the DetZero tracker on the device (sm_90a): from the all-gathered (F, K, 9) detections of S sequences to
// post-processed tracks, following tracking/tools/cfgs/tk_model_cfgs/waymo_detzero_track.yaml + tk_dataset_cfgs/waymo_dataset.yaml:
//
//   per frame   heading_process + overlap_box_filter (max_score) + transform_to_global   (datasets/data_processor.py:42-162)
//   forward     KF predict, two-stage GNN association, KF update, births, overlap_track_merge  (track_manager.py:85-216,262-310)
//   reverse     frames descending: static reverse tracks + the forward non-start entries, second stage only, merge, emit,
//               spawn (track_manager.py:109-141,218-260)
//   post        empty_track_delete (LEAST_AGE, END_REMOVE), velocity_optimize (HEADER_LENGTH), motion_classify; the shipped
//               static_drift_eliminate only rewrites trailing hit == 0 boxes, of which END_REMOVE leaves none (post_process.py)
//
// One persistent block per sequence loops over the frames in block-wide phases.  A frame's detections are staged in shared
// memory; track state, the entry pools and the association scratch live in the caller's workspace (L2-resident).
//
// Association: every (track, detection) pair is first tested on its centre distance against the sum of half-diagonals plus 0.05 m;
// a pair beyond that has BEV IoU exactly 0 (no corner lies within the 1e-2 in-box margin, no edges cross), so only near pairs go
// through bev_iou of boxgeom.cuh.  The reference's cost (1 - affinity, 5000 where cost >= 1, scipy linear_sum_assignment) makes
// the optimum a maximum-cardinality matching of the valid edges with the least total cost; that objective separates over the
// connected components of the valid-edge graph.  The components are labelled by min-hooking union-find and their edges grouped
// by root (uf_label, group_edges of assign.cuh); each one is solved exactly as a dense float64 cost matrix (double)(1.f - iou)
// by the Hungarian method with potentials (solve_dense, solve_dense_block of assign.cuh).  A component of at most SMALL_EDGES
// edges (nearly all: one detection and its track) is solved by one thread on its edges sorted by (row, column); a larger one (a
// chain of pedestrians, a crowd) by the whole block, one component at a time, with the same arithmetic and tie rule.  The dense
// cost matrix of a component lives in the per-sequence assignment scratch (SCR_CAP doubles, e.g. a 700 x 700 component).
//
// The ordered scans (the overlap filter, both merges, births) run on one thread over lists computed in parallel.
//
// Precision: the KF state is float64 once a track has had a measurement update and float32 before (as in the reference, where
// `x + K @ (z - H x)` promotes it), P / Q / K are float32, association boxes are float32 world boxes and emitted boxes float64.
// The transcendental functions and the 3x3 inverse are not those of numpy / LAPACK, so boxes agree with the numpy oracle to
// about 1e-6 relative (float32 state at km world offsets), and decisions agree wherever the oracle's margin is above rounding.
//
// Deviation: the reference's reverse pass raises KeyError when the first frames of a sequence have no track entries (frm_tracks
// is a plain dict); here such frames have no entries.
//
// Capacity: a sequence may hold max_tracks track ids and max_entries forward / reverse / output entries; the edge lists and the
// assignment scratch have fixed sizes per sequence.  Past any of them the kernel stops writing, sets overflow[s] (a bit per
// table) and the results of that sequence are invalid.
#include <float.h>
#include <limits.h>
#include "common.cuh"
#include "boxgeom.cuh"
#include "assign.cuh"
#include "eval_common.cuh"

namespace {

constexpr int NT = 512;
constexpr int EDGE_CAP = 32768;            // association edges per call
constexpr int MEDGE_CAP = 32768;           // merge edges per call
constexpr int SCR_CAP = 1 << 19;           // float64 assignment scratch per sequence
constexpr int SMALL_EDGES = 32;            // components with more edges are solved by the whole block

struct Seq {
    // track state, indexed by track id
    double *x, *size, *head, *box, *birth;  // x (T, 5), size (T, 3), head (T), box (T, 9) current bbox, birth (T, 7)
    float *P, *q, *score, *rscore;          // P (T, 25), q (T, 2), score (T), reverse score (T)
    int *cls, *hit, *first, *rhit;
    int *live, *live2, *rlive;              // forward live list (ascending ids), scratch, reverse live list (spawn order)
    // per-call scratch
    float* cbox;                            // (2T, 7) association column boxes
    int *ccls, *cref, *lab, *cnt;           // cref: column -> track id (reverse: -1 for a forward entry)
    int *e_r, *e_c, *es_r, *es_c;
    float *e_a, *es_a;
    int *m_i, *m_j, *mcnt, *moff, *madj;
    unsigned char *interesting, *dep;
    double* scr;
    // entry pools
    int *f_id, *f_hit, *f_off, *r_id, *r_hit, *r_off;
    float *f_score, *r_score;
    double* f_box;
    int *pcnt, *plo, *phi, *poff;
};

struct Shared {
    int n_live, n_rlive, next_id, n_edges, n_medges, changed, overflow, f_used, r_used, scr_used, n_rows, n_cols, n_tmp, n_births;
    int n_big;
    HungShared<NT> hs;                      // block-wide Hungarian
};

__device__ __forceinline__ double yawd(double y) {
    const double pi2 = 6.283185307179586, pi = 3.141592653589793;
    if (fabs(y) >= pi2) y = y - floor(y / pi2) * pi2;
    if (y > pi) y -= pi2;
    if (y <= -pi) y += pi2;
    return y;
}

struct Frame {                      // one frame's detections in shared memory
    float* lid;                     // (K, 7) lidar boxes after the heading filter
    float* wf;                      // (K, 7) float32 world boxes
    double* world;                  // (K, 7) float64 world boxes
    float* score;
    int* cls;
    unsigned long long* best;       // overlap filter: packed (score bits, index) of the best box of each row
    unsigned char* kept;
    int* rows;                      // association rows (detection indices)
    int* match;                     // per row: matched column or -1
    int* rcnt;                      // per component root: edge count, then offset
    int* big;                       // roots of the components solved block-wide
    int n;
};

struct Params {
    double filt[3], s1[3], s2[3], merge[3], score[3], p0, p1, q0, q1, r, dt;
    int least_age, header_len;
};

// load, heading filter and (world) transform of frame f; kept_in: the overlap filter's flags (reverse pass) or null (compute them)
__device__ void stage_frame(Frame& fr, const float* rows, int n, const double* pose, const Params& pr, unsigned char* kept_out,
                            const unsigned char* kept_in, int K) {
    fr.n = n;
    for (int i = threadIdx.x; i < n; i += NT) {
        const float* d = rows + (size_t)i * 9;
#pragma unroll
        for (int k = 0; k < 6; ++k) fr.lid[i * 7 + k] = d[k];
        fr.lid[i * 7 + 6] = yawf(d[6]);
        fr.score[i] = d[7];
        fr.cls[i] = (int)d[8];
        fr.best[i] = 0ull;
        fr.kept[i] = kept_in ? kept_in[i] : 0;
        const double x = fr.lid[i * 7], y = fr.lid[i * 7 + 1], z = fr.lid[i * 7 + 2];
        double c[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) c[r] = x * pose[r * 4] + y * pose[r * 4 + 1] + z * pose[r * 4 + 2] + pose[r * 4 + 3];
        const double h = yawd((double)fr.lid[i * 7 + 6] + atan2(pose[4], pose[0]));
        double* w = fr.world + i * 7;
        w[0] = c[0]; w[1] = c[1]; w[2] = c[2]; w[3] = fr.lid[i * 7 + 3]; w[4] = fr.lid[i * 7 + 4]; w[5] = fr.lid[i * 7 + 5]; w[6] = h;
#pragma unroll
        for (int k = 0; k < 7; ++k) fr.wf[i * 7 + k] = (float)w[k];
    }
    __syncthreads();
    if (kept_in) return;
    // overlap_box_filter: row i's set = {j : overlap(i, j) / area_i >= thr[cls_i]} (classes not masked); best = max score, the
    // later index on a tie
    for (int p = threadIdx.x; p < n * n; p += NT) {
        const int i = p / n, j = p - i * n;
        const float* a = fr.lid + i * 7;
        const float* b = fr.lid + j * 7;
        if (far_pair(a, b)) continue;
        const float ratio = bev_overlap(a, b) / (a[3] * a[4]);
        if (ratio >= (float)pr.filt[fr.cls[i] - 1])
            atomicMax(&fr.best[i], ((unsigned long long)__float_as_uint(fr.score[j]) << 32) | (unsigned)(j + 1));
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int i = 0; i < n; ++i)
            if (!fr.kept[i]) fr.kept[fr.best[i] ? (int)(fr.best[i] & 0xffffffffu) - 1 : i] = 1;
    __syncthreads();
    for (int i = threadIdx.x; i < K; i += NT) kept_out[i] = i < n ? fr.kept[i] : 0;
}

__device__ void set_overflow(Shared& sh, int bit) { atomicOr(&sh.overflow, bit); }

// GNN association of fr.rows[0..n_rows) against the columns sq.cbox[0..n_cols); fr.match[r] = column or -1
__device__ void associate(Frame& fr, Seq& sq, Shared& sh, int n_rows, int n_cols, const double* thr) {
    for (int r = threadIdx.x; r < max(n_rows, fr.n); r += NT) { fr.match[r] = -1; fr.rcnt[r] = 0; }
    for (int v = threadIdx.x; v < n_rows + n_cols; v += NT) sq.lab[v] = v;
    if (threadIdx.x == 0) { sh.n_edges = 0; sh.scr_used = 0; }
    __syncthreads();
    if (n_rows == 0 || n_cols == 0) return;
    const long long pairs = (long long)n_rows * n_cols;
    for (long long p = threadIdx.x; p < pairs; p += NT) {
        const int r = (int)(p / n_cols), c = (int)(p - (long long)r * n_cols);
        const int d = fr.rows[r];
        if (sq.ccls[c] != fr.cls[d]) continue;
        const float* a = sq.cbox + (size_t)c * 7;
        const float* b = fr.wf + d * 7;
        if (far_pair(a, b)) continue;
        const float iou = bev_iou(a, b);
        if (!(iou >= (float)thr[sq.ccls[c] - 1])) continue;
        const int e = atomicAdd(&sh.n_edges, 1);
        if (e < EDGE_CAP) { sq.e_r[e] = r; sq.e_c[e] = c; sq.e_a[e] = iou; } else set_overflow(sh, 4);
    }
    __syncthreads();
    const int ne = min(sh.n_edges, EDGE_CAP);
    if (ne == 0) return;
    uf_label<NT>(sq.lab, ne, [&](int e) { return sq.e_r[e]; }, [&](int e) { return n_rows + sq.e_c[e]; }, sh.changed);
    group_edges<NT>(sq.lab, ne, n_rows, fr.rcnt, sq.e_r, sq.e_c, sq.e_a, sq.es_r, sq.es_c, sq.es_a);
    volatile int* lab = sq.lab;
    // cost (double)(1.f - iou), 5000 off the valid edges; a chosen pair is a match when its cost is below 1
    for (int root = threadIdx.x; root < n_rows; root += NT) {
        const int end = fr.rcnt[root], beg = root ? fr.rcnt[root - 1] : 0;
        if (end == beg || uf_find(lab, root) != root) continue;
        int* er = sq.es_r + beg;
        int* ec = sq.es_c + beg;
        float* ea = sq.es_a + beg;
        const int m = end - beg;
        if (m == 1) { fr.match[er[0]] = ec[0]; continue; }
        if (m > SMALL_EDGES) continue;                              // solved block-wide below
        sort_edges(er, ec, ea, m);
        const int need = 3 * m + 8;                                 // rows and columns lists, in doubles (ints fit)
        const int base = atomicAdd(&sh.scr_used, need);
        if (base + need > SCR_CAP) { set_overflow(sh, 8); continue; }
        int* cols = (int*)(sq.scr + base);                          // distinct columns, ascending
        int nc = 0;
        for (int i = 0; i < m; ++i) {
            const int c = ec[i];
            int j = nc - 1;
            while (j >= 0 && cols[j] > c) --j;
            if (j >= 0 && cols[j] == c) continue;
            for (int k = nc; k > j + 1; --k) cols[k] = cols[k - 1];
            cols[j + 1] = c; ++nc;
        }
        int* rows = cols + nc;                                      // distinct rows (sorted already)
        int nr = 0;
        for (int i = 0; i < m; ++i) if (i == 0 || er[i] != er[i - 1]) rows[nr++] = er[i];
        const int need2 = (int)hungarian_scratch(nr, nc);
        const int base2 = atomicAdd(&sh.scr_used, need2);
        if (base2 + need2 > SCR_CAP) { set_overflow(sh, 8); continue; }
        solve_dense(nr, nc, m, [&](int i, int& ri, int& ci, double& cost) {
            ri = 0; ci = 0;
            while (rows[ri] != er[i]) ++ri;
            while (cols[ci] != ec[i]) ++ci;
            cost = (double)(1.f - ea[i]);
            return true;
        }, 5000., 1., sq.scr + base2, [&](int ri, int ci) { fr.match[rows[ri]] = cols[ci]; });
    }
    __syncthreads();
    // large components (a chain of pedestrians, a crowd): one at a time, the whole block on each
    const int nbig = block_compact(n_rows, [&](int r) {
        const int m = fr.rcnt[r] - (r ? fr.rcnt[r - 1] : 0);
        return m > SMALL_EDGES && uf_find(lab, r) == r; }, [&](int r, int pos) { fr.big[pos] = r; });
    for (int b = 0; b < nbig; ++b) {
        const int root = fr.big[b], end = fr.rcnt[root], beg = root ? fr.rcnt[root - 1] : 0;
        const int base = sh.scr_used;                               // the small components' scratch stays untouched
        int* rmap = (int*)(sq.scr + base);                          // detection row -> local row, column -> local column
        int* cmap = rmap + n_rows;
        int* rlist = cmap + n_cols;
        int* clist = rlist + n_rows;
        const int nr = block_compact(n_rows, [&](int r) { return uf_find(lab, r) == root; },
                                     [&](int r, int pos) { rmap[r] = pos; rlist[pos] = r; });
        const int nc = block_compact(n_cols, [&](int c) { return uf_find(lab, n_rows + c) == root; },
                                     [&](int c, int pos) { cmap[c] = pos; clist[pos] = c; });
        const size_t a0 = base + (size_t)(2 * n_rows + 2 * n_cols + 1) / 2 + 1;
        if (a0 + hungarian_scratch(nr, nc) > (size_t)SCR_CAP) {
            if (threadIdx.x == 0) set_overflow(sh, 8);
            __syncthreads();
            continue;
        }
        solve_dense_block<NT>(nr, nc, end - beg, [&](int i, int& ri, int& ci, double& cost) {
            ri = rmap[sq.es_r[beg + i]]; ci = cmap[sq.es_c[beg + i]];
            cost = (double)(1.f - sq.es_a[beg + i]);
            return true;
        }, 5000., 1., sq.scr + a0, sh.hs, [&](int ri, int ci) { fr.match[rlist[ri]] = clist[ci]; });
        __syncthreads();
    }
}

// overlap_track_merge over the list ids[0..n) with float32 boxes sq.cbox (same order) and classes sq.ccls; marks sq.dep[k]
__device__ void merge(Seq& sq, Shared& sh, const int* ids, int n, const Params& pr) {
    for (int k = threadIdx.x; k < n; k += NT) { sq.dep[k] = 0; sq.interesting[k] = 0; sq.mcnt[k] = 0; }
    if (threadIdx.x == 0) sh.n_medges = 0;
    __syncthreads();
    const long long pairs = (long long)n * n;
    for (long long p = threadIdx.x; p < pairs; p += NT) {
        const int i = (int)(p / n), j = (int)(p - (long long)i * n);
        if (i == j || sq.ccls[i] != sq.ccls[j]) continue;
        const float* a = sq.cbox + (size_t)i * 7;
        const float* b = sq.cbox + (size_t)j * 7;
        if (far_pair(a, b)) continue;
        const float ratio = bev_overlap(a, b) / (a[3] * a[4] + 1e-9f);
        if (!(ratio >= (float)pr.merge[sq.ccls[i] - 1])) continue;
        const int e = atomicAdd(&sh.n_medges, 1);
        if (e < MEDGE_CAP) { sq.m_i[e] = i; sq.m_j[e] = j; atomicAdd(&sq.mcnt[i], 1); sq.interesting[i] = 1; sq.interesting[j] = 1; }
        else set_overflow(sh, 16);
    }
    __syncthreads();
    const int ne = min(sh.n_medges, MEDGE_CAP);
    if (ne == 0) return;
    if (threadIdx.x == 0) {
        int run = 0;
        for (int k = 0; k < n; ++k) { sq.moff[k] = run; run += sq.mcnt[k]; sq.mcnt[k] = 0; }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < ne; e += NT) { const int i = sq.m_i[e]; sq.madj[sq.moff[i] + atomicAdd(&sq.mcnt[i], 1)] = sq.m_j[e]; }
    __syncthreads();
    // ordered scan over the tracks that take part in an overlap; dep doubles as "not fresh" until the end
    if (threadIdx.x == 0) {
        for (int i = 0; i < n; ++i) {
            if (!sq.interesting[i] || sq.dep[i]) continue;
            int best = i;
            const int* adj = sq.madj + sq.moff[i];
            for (int k = 0; k < sq.mcnt[i]; ++k) { const int j = adj[k]; if (!sq.dep[j] && ids[j] < ids[best]) best = j; }
            sq.dep[i] = 1;
            for (int k = 0; k < sq.mcnt[i]; ++k) if (!sq.dep[adj[k]]) sq.dep[adj[k]] = 1;
            sq.dep[best] = 2;                                       // kept (never fresh again)
        }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < n; k += NT) sq.dep[k] = sq.dep[k] == 1;
    __syncthreads();
}

__device__ void kf_predict(Seq& sq, int id, const Params& pr, double dt) {
    double* x = sq.x + (size_t)id * 5;
    const double* sz = sq.size + (size_t)id * 3;
    if (sq.cls[id] == 1) {
        const double speed = sqrt(x[3] * x[3] + x[4] * x[4]), lim = fmax(fmax(sz[0], sz[1]), sz[2]) / 2.;
        if (speed <= lim) { x[3] = 0.; x[4] = 0.; }
    }
    const float dtf = (float)dt;
    x[0] += (double)dtf * x[3];
    x[1] += (double)dtf * x[4];
    float* P = sq.P + (size_t)id * 25;
    float A[25];
#pragma unroll
    for (int r = 0; r < 5; ++r)
#pragma unroll
        for (int c = 0; c < 5; ++c) A[r * 5 + c] = P[r * 5 + c] + (r < 2 ? dtf * P[(r + 3) * 5 + c] : 0.f);     // F P
    float* q = sq.q + (size_t)id * 2;
#pragma unroll
    for (int r = 0; r < 5; ++r)
#pragma unroll
        for (int c = 0; c < 5; ++c) P[r * 5 + c] = A[r * 5 + c] + (c < 2 ? dtf * A[r * 5 + c + 3] : 0.f) + (r == c ? q[r < 3 ? 0 : 1] : 0.f);
    q[0] *= 1.5f; q[1] *= 1.5f;
    sq.hit[id] = 0;
    double* b = sq.box + (size_t)id * 9;
    b[0] = x[0]; b[1] = x[1]; b[2] = x[2]; b[3] = sz[0]; b[4] = sz[1]; b[5] = sz[2]; b[6] = sq.head[id]; b[7] = x[3]; b[8] = x[4];
}

__device__ void kf_update(Seq& sq, int id, const double* z, const Params& pr) {
    float* P = sq.P + (size_t)id * 25;
    const float rr = (float)pr.r;
    // S = H P H^T + R and its inverse, rounded to float32 like np.linalg.inv on float32.  The cofactors are formed in float64: Q grows
    // by 1.5x per frame, and at ~1e19 after 100 frames their float32 products would overflow
    const double s00 = (double)(P[0] + rr), s01 = P[1], s02 = P[2], s10 = P[5], s11 = (double)(P[6] + rr), s12 = P[7], s20 = P[10],
                 s21 = P[11], s22 = (double)(P[12] + rr);
    const double c00 = s11 * s22 - s12 * s21, c01 = s02 * s21 - s01 * s22, c02 = s01 * s12 - s02 * s11;
    const double c10 = s12 * s20 - s10 * s22, c11 = s00 * s22 - s02 * s20, c12 = s02 * s10 - s00 * s12;
    const double c20 = s10 * s21 - s11 * s20, c21 = s01 * s20 - s00 * s21, c22 = s00 * s11 - s01 * s10;
    const double det = s00 * c00 + s01 * c10 + s02 * c20;
    const float iS[9] = {(float)(c00 / det), (float)(c01 / det), (float)(c02 / det), (float)(c10 / det), (float)(c11 / det),
                         (float)(c12 / det), (float)(c20 / det), (float)(c21 / det), (float)(c22 / det)};
    float K[15];
#pragma unroll
    for (int r = 0; r < 5; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) K[r * 3 + c] = P[r * 5] * iS[c] + P[r * 5 + 1] * iS[3 + c] + P[r * 5 + 2] * iS[6 + c];
    double* x = sq.x + (size_t)id * 5;
    const double res[3] = {z[0] - x[0], z[1] - x[1], z[2] - x[2]};
#pragma unroll
    for (int r = 3; r < 5; ++r) x[r] += (double)K[r * 3] * res[0] + (double)K[r * 3 + 1] * res[1] + (double)K[r * 3 + 2] * res[2];
    float NP[25];
#pragma unroll
    for (int r = 0; r < 5; ++r)
#pragma unroll
        for (int c = 0; c < 5; ++c) NP[r * 5 + c] = P[r * 5 + c] - (K[r * 3] * P[c] + K[r * 3 + 1] * P[5 + c] + K[r * 3 + 2] * P[10 + c]);
#pragma unroll
    for (int k = 0; k < 25; ++k) P[k] = NP[k];
    x[0] = z[0]; x[1] = z[1]; x[2] = z[2];
    double* sz = sq.size + (size_t)id * 3;
    sz[0] = z[3]; sz[1] = z[4]; sz[2] = z[5];
    sq.head[id] = z[6];
    double* b = sq.box + (size_t)id * 9;
#pragma unroll
    for (int k = 0; k < 7; ++k) b[k] = z[k];
    b[7] = x[3]; b[8] = x[4];
}

__device__ void kf_birth(Seq& sq, int id, const double* w, int cls, float score, int f, const Params& pr) {
    double* x = sq.x + (size_t)id * 5;
    double* b = sq.box + (size_t)id * 9;
    for (int k = 0; k < 7; ++k) { b[k] = (double)(float)w[k]; sq.birth[(size_t)id * 7 + k] = b[k]; }
    b[7] = b[8] = 0.;
    x[0] = b[0]; x[1] = b[1]; x[2] = b[2]; x[3] = x[4] = 0.;
    sq.size[(size_t)id * 3] = w[3]; sq.size[(size_t)id * 3 + 1] = w[4]; sq.size[(size_t)id * 3 + 2] = w[5];
    sq.head[id] = w[6];
    float* P = sq.P + (size_t)id * 25;
    for (int k = 0; k < 25; ++k) P[k] = 0.f;
    for (int k = 0; k < 5; ++k) P[k * 6] = (float)(k < 3 ? pr.p0 : pr.p1);
    sq.q[(size_t)id * 2] = (float)pr.q0; sq.q[(size_t)id * 2 + 1] = (float)pr.q1;
    sq.cls[id] = cls; sq.score[id] = score; sq.hit[id] = 1; sq.first[id] = f;
}

__device__ void box_to_col(Seq& sq, int c, const double* b, int cls, int ref) {
#pragma unroll
    for (int k = 0; k < 7; ++k) sq.cbox[(size_t)c * 7 + k] = (float)b[k];
    sq.ccls[c] = cls;
    sq.cref[c] = ref;
}

}  // namespace

struct DzTrackOut {
    int *trk;                 // (S, T, 6): id, class, first frame, entry count, state (1 dynamic), entry offset
    int* n_tracks;            // (S)
    double* ent_box;          // (S, E, 9)
    float* ent_score;         // (S, E)
    int *ent_hit, *ent_frame; // (S, E)
    unsigned char* kept;      // (S, F, K)
    int* overflow;            // (S)
};

// one sequence's workspace; carved from a null base it only sizes it (seq_ws_bytes)
__host__ __device__ Seq carve(DzCarve& c, int F, int K, int T, int E) {
    Seq s;
    s.x = c.take<double>((size_t)T * (5 + 3 + 1 + 9 + 7));
    s.size = s.x + (size_t)T * 5; s.head = s.size + (size_t)T * 3; s.box = s.head + T; s.birth = s.box + (size_t)T * 9;
    s.P = c.take<float>((size_t)T * (25 + 2 + 2));
    s.q = s.P + (size_t)T * 25; s.score = s.q + (size_t)T * 2; s.rscore = s.score + T;
    s.cls = c.take<int>((size_t)T * 4); s.hit = s.cls + T; s.first = s.hit + T; s.rhit = s.first + T;
    s.live = c.take<int>((size_t)T * 3); s.live2 = s.live + T; s.rlive = s.live2 + T;
    s.cbox = c.take<float>((size_t)2 * T * 7);
    s.ccls = c.take<int>((size_t)2 * T * 2); s.cref = s.ccls + 2 * T;
    s.lab = c.take<int>((size_t)K + 2 * T);
    s.cnt = c.take<int>(1);
    s.e_r = c.take<int>((size_t)EDGE_CAP * 6);
    s.e_c = s.e_r + EDGE_CAP; s.es_r = s.e_c + EDGE_CAP; s.es_c = s.es_r + EDGE_CAP;
    s.e_a = (float*)(s.es_c + EDGE_CAP); s.es_a = s.e_a + EDGE_CAP;
    s.m_i = c.take<int>((size_t)MEDGE_CAP * 3); s.m_j = s.m_i + MEDGE_CAP; s.madj = s.m_j + MEDGE_CAP;
    s.mcnt = c.take<int>((size_t)2 * T * 2); s.moff = s.mcnt + 2 * T;
    s.interesting = c.take<unsigned char>((size_t)2 * T * 2); s.dep = s.interesting + 2 * T;
    s.scr = c.take<double>(SCR_CAP);
    s.f_box = (double*)c.take<char>((size_t)E * (4 + 4 + 4 + 72));
    s.f_id = (int*)(s.f_box + (size_t)E * 9); s.f_hit = s.f_id + E; s.f_score = (float*)(s.f_hit + E);
    s.f_off = c.take<int>((size_t)F + 1);
    s.r_id = c.take<int>((size_t)E * 3); s.r_hit = s.r_id + E; s.r_score = (float*)(s.r_hit + E);
    s.r_off = c.take<int>((size_t)F + 1);
    s.pcnt = c.take<int>((size_t)T * 4); s.plo = s.pcnt + T; s.phi = s.plo + T; s.poff = s.phi + T;
    return s;
}

static size_t seq_ws_bytes(int F, int K, int T, int E) {
    DzCarve c(nullptr);
    carve(c, F, K, T, E);
    return c.bytes + 256;
}

__global__ void __launch_bounds__(NT, 1)
k_track_sequences(const float* __restrict__ boxes, const int* __restrict__ counts, const int* __restrict__ num_frames,
                  const double* __restrict__ poses, int F, int K, Params pr, int T, int E, DzTrackOut out, char* ws, size_t seq_bytes) {
    const int s = blockIdx.x;
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ Shared sh;
    Frame fr;
    {
        unsigned char* p = smem;
        fr.world = (double*)p; p += (size_t)K * 7 * 8;
        fr.best = (unsigned long long*)p; p += (size_t)K * 8;
        fr.lid = (float*)p; p += (size_t)K * 7 * 4;
        fr.wf = (float*)p; p += (size_t)K * 7 * 4;
        fr.score = (float*)p; p += (size_t)K * 4;
        fr.cls = (int*)p; p += (size_t)K * 4;
        fr.rows = (int*)p; p += (size_t)K * 4;
        fr.match = (int*)p; p += (size_t)K * 4;
        fr.rcnt = (int*)p; p += (size_t)K * 4;
        fr.big = (int*)p; p += (size_t)K * 4;
        fr.kept = p;
    }
    DzCarve wc(ws + (size_t)s * seq_bytes);
    Seq sq = carve(wc, F, K, T, E);
    const int Fs = min(max(num_frames[s], 0), F);
    if (threadIdx.x == 0) {
        sh.n_live = sh.n_rlive = sh.next_id = 0; sh.overflow = 0; sh.f_used = sh.r_used = 0;
    }
    __syncthreads();
    // ---------------------------------------------------------------- forward
    for (int f = 0; f < Fs; ++f) {
        const int n = min(max(counts[(size_t)s * F + f], 0), K);
        stage_frame(fr, boxes + ((size_t)s * F + f) * K * 9, n, poses + ((size_t)s * F + f) * 16, pr,
                    out.kept + ((size_t)s * F + f) * K, nullptr, K);
        const int nl = sh.n_live;
        for (int k = threadIdx.x; k < nl; k += NT) {
            const int id = sq.live[k];
            kf_predict(sq, id, pr, pr.dt);
            box_to_col(sq, k, sq.box + (size_t)id * 9, sq.cls[id], id);
        }
        // rows: the kept detections with score >= SCORE_THRESHOLD (all of them when there is no track)
        if (threadIdx.x == 0) {
            int nr = 0;
            for (int i = 0; i < n; ++i)
                if (fr.kept[i] && (nl == 0 || (double)fr.score[i] >= pr.score[fr.cls[i] - 1])) fr.rows[nr++] = i;
            sh.n_rows = nr;
        }
        __syncthreads();
        const int nr1 = sh.n_rows;
        associate(fr, sq, sh, nl ? nr1 : 0, nl, pr.s1);
        for (int r = threadIdx.x; r < nr1; r += NT) {
            const int c = fr.match[r];
            if (c < 0) continue;
            const int id = sq.live[c], d = fr.rows[r];
            kf_update(sq, id, fr.world + d * 7, pr);
            sq.cls[id] = fr.cls[d]; sq.score[id] = fr.score[d]; sq.hit[id] = 1;
            sq.ccls[c] = -1;                                          // matched: not a stage-2 column
        }
        __syncthreads();
        // births (row order) -> fr.rcnt as a list; then stage 2 on the low-score rows and the unmatched tracks
        if (threadIdx.x == 0) {
            int nb = 0;
            for (int r = 0; r < nr1; ++r) if (fr.match[r] < 0) fr.rcnt[nb++] = fr.rows[r];
            sh.n_births = nb;
            int nr = 0;
            for (int i = 0; i < n; ++i) if (fr.kept[i] && !((double)fr.score[i] >= pr.score[fr.cls[i] - 1])) fr.rows[nr++] = i;
            sh.n_rows = nl ? nr : 0;
        }
        __syncthreads();
        const int nb = sh.n_births;
        const int id0 = sh.next_id;
        const int nbk = min(nb, T - id0);                             // births past max_tracks are dropped (overflow bit 1)
        for (int b = threadIdx.x; b < nbk; b += NT) sq.live2[b] = fr.rcnt[b];       // park the birth list
        __syncthreads();
        const int nc2 = block_compact(nl, [&](int k) { return sq.ccls[k] >= 0; },
                                      [&](int k, int pos) { sq.mcnt[pos] = k; });
        // mcnt holds the live positions of the stage-2 columns; copy their boxes into column slots nl..nl+nc2
        for (int k = threadIdx.x; k < nc2; k += NT) {
            const int c = sq.mcnt[k], id = sq.live[c];
            box_to_col(sq, nl + k, sq.box + (size_t)id * 9, sq.cls[id], id);
        }
        __syncthreads();
        {
            // associate reads columns from 0: shift the view
            Seq sv = sq;
            sv.cbox = sq.cbox + (size_t)nl * 7; sv.ccls = sq.ccls + nl; sv.cref = sq.cref + nl;
            associate(fr, sv, sh, sh.n_rows, nc2, pr.s2);
            const int nr2 = sh.n_rows;
            for (int r = threadIdx.x; r < nr2; r += NT) {
                const int c = fr.match[r];
                if (c < 0) continue;
                const int id = sv.cref[c];
                sq.hit[id] = 2; sq.score[id] = fr.score[fr.rows[r]];
            }
        }
        __syncthreads();
        if (threadIdx.x == 0 && nbk < nb) set_overflow(sh, 1);
        for (int b = threadIdx.x; b < nbk; b += NT) {
            const int d = sq.live2[b];
            kf_birth(sq, id0 + b, fr.world + d * 7, fr.cls[d], fr.score[d], f, pr);
            sq.live[nl + b] = id0 + b;
        }
        __syncthreads();
        if (threadIdx.x == 0) { sh.next_id = id0 + nbk; sh.n_live = nl + nbk; }
        __syncthreads();
        const int nl2 = sh.n_live;
        for (int k = threadIdx.x; k < nl2; k += NT) { const int id = sq.live[k]; box_to_col(sq, k, sq.box + (size_t)id * 9, sq.cls[id], id); }
        __syncthreads();
        merge(sq, sh, sq.live, nl2, pr);
        const int nl3 = block_compact(nl2, [&](int k) { return !sq.dep[k]; }, [&](int k, int pos) { sq.live2[pos] = sq.live[k]; });
        // emit the forward entries of this frame
        const int base = sh.f_used;
        const int ne = min(nl3, E - base);
        for (int k = threadIdx.x; k < nl3; k += NT) {
            const int id = sq.live2[k];
            sq.live[k] = id;
            if (k >= ne) continue;
            const int e = base + k;
            sq.f_id[e] = id; sq.f_hit[e] = sq.hit[id]; sq.f_score[e] = sq.score[id];
            for (int j = 0; j < 9; ++j) sq.f_box[(size_t)e * 9 + j] = sq.box[(size_t)id * 9 + j];
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            if (ne < nl3) set_overflow(sh, 2);
            sq.f_off[f] = base; sh.f_used = base + ne; sh.n_live = nl3;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) sq.f_off[Fs] = sh.f_used;
    __syncthreads();
    // ---------------------------------------------------------------- reverse
    for (int f = Fs - 1; f >= 0; --f) {
        const int n = min(max(counts[(size_t)s * F + f], 0), K);
        stage_frame(fr, boxes + ((size_t)s * F + f) * K * 9, n, poses + ((size_t)s * F + f) * 16, pr, nullptr,
                    out.kept + ((size_t)s * F + f) * K, K);
        const int nrv = sh.n_rlive, eb = sq.f_off[f], ee = sq.f_off[f + 1];
        for (int k = threadIdx.x; k < nrv; k += NT) {
            const int id = sq.rlive[k];
            sq.rhit[id] = 0;                                          // a reverse track never moves (zero velocity)
            box_to_col(sq, k, sq.birth + (size_t)id * 7, sq.cls[id], id);
        }
        const int nfc = block_compact(ee - eb, [&](int k) { return sq.first[sq.f_id[eb + k]] != f; },
                                      [&](int k, int pos) {
                                          const int e = eb + k;
                                          box_to_col(sq, nrv + pos, sq.f_box + (size_t)e * 9, sq.cls[sq.f_id[e]], -1);
                                      });
        if (threadIdx.x == 0) {
            int nr = 0;
            for (int i = 0; i < n; ++i) if (fr.kept[i] && !((double)fr.score[i] >= pr.score[fr.cls[i] - 1])) fr.rows[nr++] = i;
            sh.n_rows = nr;
        }
        __syncthreads();
        const int nr = sh.n_rows;
        associate(fr, sq, sh, nr, nrv + nfc, pr.s2);
        for (int r = threadIdx.x; r < nr; r += NT) {
            const int c = fr.match[r];
            if (c < 0 || c >= nrv) continue;
            const int id = sq.cref[c];
            sq.rhit[id] = 2; sq.rscore[id] = fr.score[fr.rows[r]];
        }
        __syncthreads();
        merge(sq, sh, sq.rlive, nrv, pr);
        const int nrv2 = block_compact(nrv, [&](int k) { return !sq.dep[k]; }, [&](int k, int pos) { sq.live2[pos] = sq.rlive[k]; });
        const int base = sh.r_used;
        const int ne = min(nrv2, E - base);
        for (int k = threadIdx.x; k < nrv2; k += NT) {
            const int id = sq.live2[k];
            sq.rlive[k] = id;
            if (k < ne) { sq.r_id[base + k] = id; sq.r_hit[base + k] = sq.rhit[id]; sq.r_score[base + k] = sq.rscore[id]; }
        }
        __syncthreads();
        // spawn a reverse track for every forward track that starts here (entry order = id order)
        const int nsp = block_compact(ee - eb, [&](int k) { return sq.first[sq.f_id[eb + k]] == f; },
                                      [&](int k, int pos) {
                                          const int e = eb + k, id = sq.f_id[e];
                                          sq.rlive[nrv2 + pos] = id; sq.rscore[id] = sq.f_score[e]; sq.rhit[id] = 1;
                                      });
        if (threadIdx.x == 0) {
            if (ne < nrv2) set_overflow(sh, 2);
            sq.r_off[f] = base; sh.r_used = base + ne; sh.n_rlive = nrv2 + nsp;
        }
        __syncthreads();
    }
    // ---------------------------------------------------------------- post-processing
    const int nid = sh.next_id, nf = sh.f_used, nrr = sh.r_used;
    for (int id = threadIdx.x; id < nid; id += NT) { sq.pcnt[id] = 0; sq.plo[id] = INT_MAX; sq.phi[id] = -1; }
    __syncthreads();
    for (int f = 0; f < Fs; ++f) {                               // frame of every pooled entry: from the frame offsets
        const int fb = sq.f_off[f], fe = f + 1 < Fs ? sq.f_off[f + 1] : nf;
        for (int e = fb + threadIdx.x; e < fe; e += NT)
            if (sq.f_hit[e] > 0) { const int id = sq.f_id[e]; atomicAdd(&sq.pcnt[id], 1); atomicMin(&sq.plo[id], f); atomicMax(&sq.phi[id], f); }
        const int rb = sq.r_off[f], re = f > 0 ? sq.r_off[f - 1] : nrr;
        for (int e = rb + threadIdx.x; e < re; e += NT)
            if (sq.r_hit[e] > 0) { const int id = sq.r_id[e]; atomicAdd(&sq.pcnt[id], 1); atomicMin(&sq.plo[id], f); atomicMax(&sq.phi[id], f); }
    }
    __syncthreads();
    int* trk = out.trk + (size_t)s * T * 6;
    if (threadIdx.x == 0) sh.n_tmp = 0;
    __syncthreads();
    // surviving ids in id order; their entry offsets by a running sum (thread 0 handles the scan over the compacted list)
    const int nsurv = block_compact(nid, [&](int id) { return sq.pcnt[id] >= pr.least_age; },
                                    [&](int id, int pos) { sq.poff[pos] = id; });
    if (threadIdx.x == 0) {
        int run = 0;
        for (int k = 0; k < nsurv; ++k) {
            const int id = sq.poff[k], cnt = sq.phi[id] - sq.plo[id] + 1;
            int* t = trk + (size_t)k * 6;
            t[0] = id; t[1] = sq.cls[id]; t[2] = sq.plo[id]; t[3] = cnt; t[4] = 0; t[5] = run;
            sq.pcnt[id] = run;                                   // pcnt becomes the entry offset of a survivor
            run += cnt;
        }
        if (run > E) set_overflow(sh, 2);
        out.n_tracks[s] = run > E ? 0 : nsurv;
        sh.n_tmp = run > E ? 0 : nsurv;
    }
    __syncthreads();
    const int nt = sh.n_tmp;
    for (int k = threadIdx.x; k < nid; k += NT) sq.live2[k] = -1;
    __syncthreads();
    for (int k = threadIdx.x; k < nt; k += NT) sq.live2[trk[(size_t)k * 6]] = k;           // id -> survivor index
    __syncthreads();
    double* obox = out.ent_box + (size_t)s * E * 9;
    float* oscore = out.ent_score + (size_t)s * E;
    int* ohit = out.ent_hit + (size_t)s * E;
    int* oframe = out.ent_frame + (size_t)s * E;
    for (int f = 0; f < Fs; ++f) {
        const int fb = sq.f_off[f], fe = f + 1 < Fs ? sq.f_off[f + 1] : nf;
        for (int e = fb + threadIdx.x; e < fe; e += NT) {
            const int id = sq.f_id[e], k = sq.live2[id];
            if (k < 0 || f < sq.plo[id] || f > sq.phi[id]) continue;
            const int o = sq.pcnt[id] + f - sq.plo[id];
            for (int j = 0; j < 9; ++j) obox[(size_t)o * 9 + j] = sq.f_box[(size_t)e * 9 + j];
            oscore[o] = sq.f_score[e]; ohit[o] = sq.f_hit[e]; oframe[o] = f;
        }
        const int rb = sq.r_off[f], re = f > 0 ? sq.r_off[f - 1] : nrr;
        for (int e = rb + threadIdx.x; e < re; e += NT) {
            const int id = sq.r_id[e], k = sq.live2[id];
            if (k < 0 || f < sq.plo[id] || f > sq.phi[id]) continue;
            const int o = sq.pcnt[id] + f - sq.plo[id];
            for (int j = 0; j < 7; ++j) obox[(size_t)o * 9 + j] = sq.birth[(size_t)id * 7 + j];
            obox[(size_t)o * 9 + 7] = 0.; obox[(size_t)o * 9 + 8] = 0.;
            oscore[o] = sq.r_score[e]; ohit[o] = sq.r_hit[e]; oframe[o] = f;
        }
    }
    __syncthreads();
    // velocity_optimize: finite differences over the first HEADER_LENGTH entries
    for (int k = threadIdx.x; k < nt; k += NT) {
        const int cnt = trk[(size_t)k * 6 + 3], o = trk[(size_t)k * 6 + 5];
        const int pl = cnt > pr.header_len ? pr.header_len : cnt - 1;
        for (int j = 0; j < pl; ++j) {
            double* b = obox + (size_t)(o + j) * 9;
            b[7] = (b[9] - b[0]) * 10.;
            b[8] = (b[10] - b[1]) * 10.;
        }
    }
    __syncthreads();
    // motion_classify: dynamic if any pair of hit == 1 boxes overlaps by <= 1e-4 (a far pair overlaps by exactly 0)
    for (int k = 0; k < nt; ++k) {
        const int cnt = trk[(size_t)k * 6 + 3], o = trk[(size_t)k * 6 + 5];
        if (threadIdx.x == 0) sh.changed = 0;
        __syncthreads();
        for (int p = threadIdx.x; p < cnt * cnt; p += NT) {
            const int a = p / cnt, b = p - a * cnt;
            if (ohit[o + a] != 1 || ohit[o + b] != 1 || sh.changed) continue;
            float ba[7], bb[7];
            for (int j = 0; j < 7; ++j) { ba[j] = (float)obox[(size_t)(o + a) * 9 + j]; bb[j] = (float)obox[(size_t)(o + b) * 9 + j]; }
            if (far_pair(ba, bb) || bev_overlap(ba, bb) <= 1e-4f) sh.changed = 1;
        }
        __syncthreads();
        int hits = 0;
        if (threadIdx.x == 0) {
            for (int j = 0; j < cnt; ++j) hits += ohit[o + j] == 1;
            trk[(size_t)k * 6 + 4] = hits >= 2 && sh.changed;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) out.overflow[s] = sh.overflow;
}

static size_t track_smem(int K) { return (size_t)K * (7 * 8 + 8 + 7 * 4 * 2 + 4 * 6) + K + 16; }

extern "C" size_t dz_track_sequences_ws_bytes(int S, int F, int K, int max_tracks, int max_entries) {
    return (size_t)S * dz_align_up(seq_ws_bytes(F, K, max_tracks, max_entries), 256) + 256;
}

extern "C" int dz_track_sequences(const float* boxes, const int* counts, const int* num_frames, const double* poses, int S, int F, int K,
                                  const double* params, int max_tracks, int max_entries, int* trk, int* n_tracks, double* ent_box,
                                  float* ent_score, int* ent_hit, int* ent_frame, unsigned char* kept, int* overflow, void* ws,
                                  size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(boxes && counts && num_frames && poses && params && trk && n_tracks && ent_box && ent_score && ent_hit && ent_frame &&
                 kept && overflow && ws && S >= 0 && F >= 1 && K >= 1 && K <= 512 && max_tracks >= 1 && max_entries >= 1);
    if (S == 0) return DZ_OK;
    if (ws_bytes < dz_track_sequences_ws_bytes(S, F, K, max_tracks, max_entries)) {
        dz_set_error("dz_track_sequences: workspace too small");
        return DZ_ERR_WORKSPACE;
    }
    Params pr;
    for (int c = 0; c < 3; ++c) {
        pr.filt[c] = params[c]; pr.s1[c] = params[3 + c]; pr.s2[c] = params[6 + c]; pr.merge[c] = params[9 + c]; pr.score[c] = params[12 + c];
    }
    pr.p0 = params[15]; pr.p1 = params[16]; pr.q0 = params[17]; pr.q1 = params[18]; pr.r = params[19]; pr.dt = params[20];
    pr.least_age = (int)params[21]; pr.header_len = (int)params[22];
    DzTrackOut out{trk, n_tracks, ent_box, ent_score, ent_hit, ent_frame, kept, overflow};
    const size_t smem = track_smem(K);
    DZ_CUDA(cudaFuncSetAttribute(k_track_sequences, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const size_t seq_bytes = dz_align_up(seq_ws_bytes(F, K, max_tracks, max_entries), 256);
    char* base = (char*)dz_align_up((size_t)ws, 256);
    k_track_sequences<<<S, NT, smem, (cudaStream_t)stream>>>(boxes, counts, num_frames, poses, F, K, pr, max_tracks, max_entries, out,
                                                             base, seq_bytes);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

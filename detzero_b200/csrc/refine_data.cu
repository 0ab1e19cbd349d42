// refine_data.cu -- refiner inputs on the device (SURVEY.md §8f row 2, "fused with refiner input encoding"), sm_90a.
//
// From collated frames (rows [b, x, y, z, tanh(i), ...] of io.prepare_points / FramePipeline, frame_offsets), float64 poses and
// float64 world track boxes, build what PositionTransformer / GeometryTransformer / ConfidencePointnet consume, and map refined boxes
// back to each frame.  Replaces, per track, the host numpy of
//   daemon/prepare_object_data.py:241-327                 crop of every box's (enlarged) points from its frame
//   refining/detzero_refine/utils/data_utils.py:12-30     sample_points
//   waymo_position_dataset.py:31-184                      PRM: init-box frame, 256 query + 48 memory points per box, [xyz, i, p2co, score (, class)]
//   waymo_confidence_dataset.py:59-162                    CRM: the same frame, 256 points per box
//   waymo_geometry_dataset.py:26-154                      GRM: box frames, top-3 boxes as queries, 4096 memory rows [xyz, i, p2s, score]
//   waymo_position_dataset.py:257-286, waymo_geometry_dataset.py:160-186   revert_to_each_frame
//
// Passes (everything on the caller's stream, no host synchronisation, no (boxes, cap) index list):
//   prep    per box slot: the float64 transforms, the enlarged crop box, per-box outputs (trajectory, mask / conf score)
//   count   per (box, chunk of its frame): points inside the box (the in/out test of track.cu's crop, boxgeom.cuh pt_in_box3d)
//   scan    per box: exclusive prefix of its chunk counts + its total; per track: GRM offsets, top-scored query boxes
//   select  per (box, stream) and per track (GRM memory): the k ranks with the smallest keys, by an 8-bit radix select on keys that
//           are recomputed from the rank (nothing stored per candidate), then an ordered compaction -> sorted ranks
//   fill    every output row no point lands in: padded samples (encoded zero points: p2co = -corner, score, class) and padded boxes
//   write   the count pass again; each in-box point finds its rank, looks it up in the sorted selection and writes its encoded row
//
// Deliberate deviations from the reference (restated in oracle/refine_data_ref.py):
//   1. Sampling is deterministic.  Of n candidates, k are kept: the ranks with the k smallest keys
//        key(r) = mix64(base + r),  base = mix64(mix64(mix64(seed) ^ track_uid) ^ (box_slot << 8 | stream))   (mod 2^64)
//      mix64(z) = splitmix64: z += 0x9E3779B97F4A7C15; z = (z ^ z>>30) * 0xBF58476D1CE4E5B9; z = (z ^ z>>27) * 0x94D049BB133111EB;
//      z ^ z>>31.  It is a bijection, so keys are distinct; the kept ranks are sorted: a uniform k-subset in sorted order, as
//      random.sample + sort draws.  A track's inputs depend on (seed, track_uid) only, not on its batch, chunk or GPU.
//      Streams: PRM query 0, PRM memory 1, CRM 2, GRM query 3 (slot = that box), GRM memory 4 (slot 0, over the whole track).
//   2. Geometry is float64: pose, init-box and box transforms are composed per box from float64 poses and world boxes and applied
//      to the float32 lidar points; outputs are float32.  (The reference rounds its trajectory to float32: ~5e-4 m at Waymo's
//      world offsets.)
//   3. GRM's query count is min(nq, L) per track (the reference lowers self.query_num for every later track).
//   4. The crop tests each point in float64 world coordinates relative to the box centre (rounded to float32 for the shared
//      float32 test), where the reference tests float32 world points: only points within ~1e-3 m of an enlarged face can differ.
//
// Training samples (the training branch of WaymoPositionDataset / WaymoGeometryDataset / WaymoConfidenceDataset
// .extract_track_feature, with geometry_augment.py:65-77 augment_single_box for the GRM; restated in oracle/refine_train_data_ref.py,
// and for the PRM in tests/prm_train_data_ref.py):
//   crop    dz_crop_tracks runs prep / count / scan / write once and copies every in-box point row to a frame of its own (one pose
//           per box), the layout the builders read with crop = 0, so the crop leaves the epoch loop.
//   draw    k_rd_draw, one block per track, keyed on (epoch_seed(seed, epoch), track_uid) with the streams ST_TR_*:
//             eligible slots: the matched ones (PRM, GRM), every valid one (CRM); m of them
//             kept count n = lo + key mod (m - lo + 1), lo = min(5, m), key = mix64(key_base(.., 0, ST_TR_COUNT)): the bias of a
//               64-bit key reduced mod at most 200 is below 200 / 2^64 < 2^-56
//             kept: the k-subset rule of select (k = n of the m eligible ranks), in ascending slot order
//             GRM queries: min(nq, n) kept positions by the same rule; PRM / CRM init box: a kept position, key mod n (ST_TR_INIT)
//             GRM flip bits: the top bit of key(i) of ST_TR_FLIP per kept position i
//           epoch_seed(seed, epoch) = mix64(mix64(seed) + epoch); the point samples of a training build use it as their seed.
//   build   dz_refine_train_inputs (GRM, CRM) and dz_position_train_inputs (PRM) gather the kept slots into a derived track table and
//           run the passes above on it, with the drawn query positions in k_rd_track (GRM), the drawn init box in k_rd_prep (PRM,
//           CRM) and the flip applied to box-local y of the memory rows in the write pass (GRM; the query points are never flipped,
//           as the reference copies them first).  The PRM's gt_pos_trajectory is the kept ground truth taken into the drawn init
//           box's frame by k_rd_prep, through the same float64 to_init_frame as pos_trajectory (init_coords_transform: heading
//           limited to [-pi, pi) before and after the rotation).
//   The PRM build keeps deviations 1 (keyed sampling, streams 0 and 1 on the kept positions), 2 (float64 geometry) and 5 unchanged.
//   Deviation 5: the reference keeps random.sample's order of the kept boxes; here they are in ascending slot order.  Every
//   consumer is invariant to the order of a track's boxes (per-box encoders, max-pools, BatchNorm statistics, decoder attention
//   over the memory, summed losses), so no distribution the model sees changes.  The PRM decoder uses no order-dependent mask
//   (PositionHead.forward passes attn_mask = None), so its ascending order changes nothing the model sees either.
#include "common.cuh"
#include "boxgeom.cuh"
#include "refine_frame.cuh"

enum { RD_PRM = 0, RD_CRM = 1, RD_GRM = 2, RD_CROP = 3 };
enum { ST_PRM_Q = 0, ST_PRM_M = 1, ST_CRM = 2, ST_GRM_Q = 3, ST_GRM_M = 4 };
enum { ST_TR_COUNT = 5, ST_TR_KEEP = 6, ST_TR_QUERY = 7, ST_TR_INIT = 8, ST_TR_FLIP = 9 };
static constexpr int RD_CHUNK = 4096;              // points of a frame per count / write block

struct RdBox {
    double G[12];          // lidar point -> world, relative to the box centre (row-major 3x4)
    double E[12];          // -> encoding frame: init-box frame (PRM, CRM) or the box's own frame (GRM)
    double cc[27];         // PRM / CRM: the 8 corners (boxes_to_corners_3d order) + centre of the box in the init frame; GRM: dims / 2
    float crop[8];         // (0, 0, 0, enlarged dx, dy, dz, world heading)
    int p0, p1;            // the frame's point rows; p1 == p0 for padded slots
    float score;
    int pad;
};

struct RdParams {
    const float* pts; int pstride; const int* foff; int F;
    const double* poses; const double* boxes; const int* fob; const float* scores; const int* box_num; const int* cls;
    const long long* uid;
    int B, L, kind, with_class, C, kq, km, nq, qout, crop, bev; double enlarge; unsigned long long seed;
    RdBox* bx; int* cc; int n_chunks; int* n; int* goff; int* gtot; int* qidx; int* qnum; int* sel;
    float* q_pts; float* m_pts; float* traj; float* box_f; float* track_f; int* query_num;
    // training builds (NULL otherwise): drawn GRM query positions (B, nq), CRM init positions (B), GRM flip bits (B, L); the
    // derived gt_geo_trajectory (B, L, 7) f32 and gt_geo_query_boxes (B, qout, 7)
    const int* qsel; const int* init; const unsigned char* flip; const float* gt_traj; float* gt_box_f;
    // PRM training builds (NULL otherwise): the kept ground truth (B, L, 7) f64 world, and gt_pos_trajectory (B, L, 7) f32
    const double* gt_w; float* gt_pos;
    // dz_crop_tracks: the first output row of each box slot, the output rows (width C)
    const int* rbase; float* rows;
};

__host__ __device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__host__ __device__ __forceinline__ unsigned long long epoch_seed(unsigned long long seed, long long epoch) {
    return mix64(mix64(seed) + (unsigned long long)epoch);
}

__device__ __forceinline__ unsigned long long key_base(unsigned long long seed, long long uid, int slot, int stream) {
    return mix64(mix64(mix64(seed) ^ (unsigned long long)uid) ^ (((unsigned long long)slot << 8) | (unsigned long long)stream));
}

__device__ __forceinline__ int track_len(const RdParams& P, int b) { return min(max(P.box_num[b], 0), P.L); }

// rows of the selection lists
__device__ __forceinline__ int* sel_list(const RdParams& P, int b, int j, int stream) {
    if (P.kind == RD_PRM) return P.sel + ((size_t)b * P.L + j) * (P.kq + P.km) + (stream == ST_PRM_M ? P.kq : 0);
    if (P.kind == RD_CRM) return P.sel + ((size_t)b * P.L + j) * P.kq;
    const size_t base = (size_t)b * (P.nq * P.kq + P.km);                    // GRM: j = query slot, or the memory list
    return P.sel + base + (stream == ST_GRM_M ? (size_t)P.nq * P.kq : (size_t)j * P.kq);
}

// ---- prep: one thread per box slot --------------------------------------------------------------------------------------------
__global__ void k_rd_prep(RdParams P) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.B * P.L) return;
    const int b = t / P.L, j = t % P.L, L = track_len(P, b);
    RdBox& o = P.bx[t];
    if (j >= L) {
        o.p0 = o.p1 = 0;
        if (P.traj) for (int d = 0; d < 7; ++d) P.traj[(size_t)t * 7 + d] = 0.f;
        if (P.gt_pos) for (int d = 0; d < 7; ++d) P.gt_pos[(size_t)t * 7 + d] = 0.f;
        if (P.kind == RD_PRM) P.box_f[t] = 1.f;                          // padding_mask
        if (P.kind == RD_CRM) P.box_f[t] = -1.f;                         // conf_score padding
        return;
    }
    const double* bw = P.boxes + (size_t)t * 7;
    const int f = min(max(P.fob[t], 0), P.F - 1);
    const double* pose = P.poses + (size_t)f * 16;
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) o.G[r * 4 + c] = pose[r * 4 + c];
        o.G[r * 4 + 3] = pose[r * 4 + 3] - bw[r];
    }
    o.crop[0] = o.crop[1] = o.crop[2] = 0.f;
    o.crop[3] = (float)(bw[3] * P.enlarge);
    o.crop[4] = (float)(bw[4] * P.enlarge);
    o.crop[5] = P.bev ? 100.f : (float)(bw[5] * P.enlarge);
    o.crop[6] = (float)bw[6];
    o.p0 = P.foff[f];
    o.p1 = P.foff[f + 1];
    o.score = P.scores ? P.scores[t] : 0.f;
    for (int d = 0; d < 12; ++d) o.E[d] = 0.0;
    if (P.kind == RD_CROP) return;
    if (P.kind == RD_GRM) {                                              // local_coords_transform: rotate by -heading
        const double c = cos(bw[6]), s = sin(bw[6]);
        o.E[0] = c; o.E[1] = s; o.E[4] = -s; o.E[5] = c; o.E[10] = 1.0;
        for (int d = 0; d < 3; ++d) o.cc[d] = bw[3 + d] / 2;
        for (int d = 0; d < 7; ++d) P.traj[(size_t)t * 7 + d] = (float)bw[d];
        return;
    }
    // init_coords_transform: init box = traj[L // 2] (heading wrapped), or the drawn one of a training build; trajectory into its frame
    const int ii = P.init ? min(max(P.init[b], 0), L - 1) : L / 2;
    const double* bi = P.boxes + ((size_t)b * P.L + ii) * 7;
    const InitFrame fr = init_frame(bi);
    const double yi = fr.yaw, c = fr.c, s = fr.s;
    o.E[0] = c; o.E[1] = s; o.E[4] = -s; o.E[5] = c; o.E[10] = 1.0;
    double loc[7];
    to_init_frame(fr, bi, bw, loc);
    o.E[3] = loc[0]; o.E[7] = loc[1]; o.E[11] = loc[2];
    const double ch = cos(loc[6]), sh = sin(loc[6]);
    for (int k = 0; k < 8; ++k) {                                         // box_utils.boxes_to_corners_3d
        const double tx = ((k == 0 || k == 1 || k == 4 || k == 5) ? 0.5 : -0.5) * loc[3];
        const double ty = ((k == 0 || k == 3 || k == 4 || k == 7) ? 0.5 : -0.5) * loc[4];
        const double tz = (k < 4 ? -0.5 : 0.5) * loc[5];
        o.cc[k * 3 + 0] = loc[0] + tx * ch - ty * sh;
        o.cc[k * 3 + 1] = loc[1] + tx * sh + ty * ch;
        o.cc[k * 3 + 2] = loc[2] + tz;
    }
    for (int d = 0; d < 3; ++d) o.cc[24 + d] = loc[d];
    if (P.kind == RD_PRM) {
        for (int d = 0; d < 7; ++d) P.traj[(size_t)t * 7 + d] = (float)loc[d];
        if (P.gt_pos) {
            double g[7];
            to_init_frame(fr, bi, P.gt_w + (size_t)t * 7, g);
            for (int d = 0; d < 7; ++d) P.gt_pos[(size_t)t * 7 + d] = (float)g[d];
        }
        P.box_f[t] = 0.f;
        if (j == 0) {
            for (int d = 0; d < 6; ++d) P.track_f[(size_t)b * 7 + d] = (float)bi[d];
            P.track_f[(size_t)b * 7 + 6] = (float)yi;
        }
    } else {
        P.box_f[t] = o.score;
    }
}

// [xyz, intensity, p2co (27), score (, class one-hot)] of a point e (encoding frame) -- padded samples are e = 0, i = 0
__device__ __forceinline__ void emit_p2co(float* out, const double e[3], float inten, const RdBox& bx, int with_class, int cls) {
    for (int d = 0; d < 3; ++d) out[d] = (float)e[d];
    out[3] = inten;
#pragma unroll
    for (int k = 0; k < 9; ++k)
        for (int d = 0; d < 3; ++d) out[4 + k * 3 + d] = (float)(e[d] - bx.cc[k * 3 + d]);
    out[31] = bx.score;
    if (with_class)
        for (int d = 0; d < 3; ++d) out[32 + d] = (d == cls - 1) ? 1.f : 0.f;
}

__device__ __forceinline__ int find_rank(const int* list, int m, int r) {          // index of r in the sorted list, or -1
    int lo = 0, hi = m;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(list + mid) < r) lo = mid + 1; else hi = mid; }
    return (lo < m && __ldg(list + lo) == r) ? lo : -1;
}

// one in-box point of box slot t with rank r (its position among the box's points, in frame order)
__device__ void write_point(const RdParams& P, const RdBox& bx, int t, int r, int p, int qi, int goff) {
    const int b = t / P.L, j = t % P.L, n = P.n[t];
    const float* q = P.pts + (size_t)p * P.pstride;
    if (P.kind == RD_CROP) {
        float* o = P.rows + ((size_t)P.rbase[t] + r) * P.C;
        for (int d = 0; d < P.C; ++d) o[d] = q[d];
        return;
    }
    const double x = q[1], y = q[2], z = q[3];
    double g[3], e[3];
    for (int d = 0; d < 3; ++d) g[d] = bx.G[d * 4] * x + bx.G[d * 4 + 1] * y + bx.G[d * 4 + 2] * z + bx.G[d * 4 + 3];
    for (int d = 0; d < 3; ++d) e[d] = bx.E[d * 4] * g[0] + bx.E[d * 4 + 1] * g[1] + bx.E[d * 4 + 2] * g[2] + bx.E[d * 4 + 3];
    const float inten = q[4];
    if (P.kind == RD_GRM) {
        if (qi >= 0) {
            const int s = find_rank(sel_list(P, b, qi, ST_GRM_Q), min(n, P.kq), r);
            if (s >= 0) {
                float* o = P.q_pts + (((size_t)b * P.qout + qi) * P.kq + s) * 4;
                o[0] = (float)e[0]; o[1] = (float)e[1]; o[2] = (float)e[2]; o[3] = inten;
            }
        }
        if (P.flip && P.flip[t]) e[1] = -e[1];                               // augment_single_box, after the query copy
        const int s = find_rank(sel_list(P, b, 0, ST_GRM_M), min(P.gtot[b], P.km), goff + r);
        if (s >= 0) {
            float* o = P.m_pts + ((size_t)b * P.km + s) * 11;
            for (int d = 0; d < 3; ++d) {
                o[d] = (float)e[d];
                o[4 + d] = (float)(bx.cc[d] - e[d]);
                o[7 + d] = (float)(bx.cc[d] + e[d]);
            }
            o[3] = inten;
            o[10] = bx.score;
        }
        return;
    }
    const int cls = P.cls[b];
    int s = find_rank(sel_list(P, b, j, P.kind == RD_PRM ? ST_PRM_Q : ST_CRM), min(n, P.kq), r);
    if (s >= 0) emit_p2co(P.q_pts + (((size_t)b * P.L + j) * P.kq + s) * P.C, e, inten, bx, P.with_class, cls);
    if (P.kind == RD_PRM) {
        s = find_rank(sel_list(P, b, j, ST_PRM_M), min(n, P.km), r);
        if (s >= 0) emit_p2co(P.m_pts + (((size_t)b * P.L + j) * P.km + s) * P.C, e, inten, bx, P.with_class, cls);
    }
}

// ---- count (WRITE = 0) / write (WRITE = 1): block = (box slot, chunk of the box's frame) -------------------------------------
// Same structure as track.cu's k_crop: pass 1 counts per (box, chunk), pass 2 re-runs the same test and ranks each in-box point
// by the exclusive prefix of its box's chunk counts -- the same in/out decision in both passes.
template <int WRITE>
__global__ void __launch_bounds__(256) k_rd_crop(RdParams P) {
    const int t = blockIdx.x, chunk = blockIdx.y;
    __shared__ RdBox sb;
    __shared__ int s_warp[8], s_base, s_qi, s_goff;
    for (int i = threadIdx.x; i < (int)(sizeof(RdBox) / 4); i += blockDim.x) ((int*)&sb)[i] = ((const int*)(P.bx + t))[i];
    if (WRITE && threadIdx.x == 0) {
        s_base = P.cc[(size_t)t * P.n_chunks + chunk];                     // exclusive prefix (after the scan)
        const int b = t / P.L, j = t % P.L;
        s_qi = -1;
        s_goff = 0;
        if (P.kind == RD_GRM) {
            for (int i = 0; i < P.qnum[b]; ++i) if (P.qidx[b * P.nq + i] == j) s_qi = i;
            s_goff = P.goff[t];
        }
    }
    __syncthreads();
    const int lo = sb.p0 + chunk * RD_CHUNK, hi = min(sb.p1, lo + RD_CHUNK);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int run = 0;
    for (int p0 = lo; p0 < hi; p0 += 256) {
        const int p = p0 + threadIdx.x;
        bool in = false;
        if (p < hi) {
            if (P.crop) {
                const float* q = P.pts + (size_t)p * P.pstride;
                const double x = q[1], y = q[2], z = q[3];
                const float gx = (float)(sb.G[0] * x + sb.G[1] * y + sb.G[2] * z + sb.G[3]);
                const float gy = (float)(sb.G[4] * x + sb.G[5] * y + sb.G[6] * z + sb.G[7]);
                const float gz = (float)(sb.G[8] * x + sb.G[9] * y + sb.G[10] * z + sb.G[11]);
                in = pt_in_box3d(gx, gy, gz, sb.crop);
            } else {
                in = true;
            }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, in);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) { const int c = s_warp[w]; before += w < warp ? c : 0; total += c; }
        if (WRITE && in) write_point(P, sb, t, s_base + run + before + __popc(bal & ((1u << lane) - 1u)), p, s_qi, s_goff);
        run += total;
        __syncthreads();
    }
    if (!WRITE && threadIdx.x == 0) P.cc[(size_t)t * P.n_chunks + chunk] = run;
}

// ---- scan: per box, exclusive prefix of its chunk counts + the box total ---------------------------------------------------------
__global__ void k_rd_scan(RdParams P) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.B * P.L) return;
    int* c = P.cc + (size_t)t * P.n_chunks;
    int run = 0;
    for (int k = 0; k < P.n_chunks; ++k) { const int v = c[k]; c[k] = run; run += v; }
    P.n[t] = run;
}

// ---- per track: GRM offsets of each box in the concatenation, the query boxes (score descending, ties: later index first),
// ---- geo_query_boxes (dims only) and geo_query_num
__global__ void k_rd_track(RdParams P) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= P.B) return;
    const int L = track_len(P, b);
    int run = 0;
    for (int j = 0; j < L; ++j) { P.goff[(size_t)b * P.L + j] = run; run += P.n[(size_t)b * P.L + j]; }
    P.gtot[b] = run;
    const int nq = min(P.nq, L);
    int taken[8];
    for (int i = 0; i < nq; ++i) {
        if (P.qsel) { taken[i] = P.qidx[b * P.nq + i] = P.qsel[b * P.nq + i]; continue; }
        int best = -1;
        for (int j = L - 1; j >= 0; --j) {
            bool used = false;
            for (int u = 0; u < i; ++u) used |= taken[u] == j;
            if (!used && (best < 0 || P.scores[(size_t)b * P.L + j] > P.scores[(size_t)b * P.L + best])) best = j;
        }
        taken[i] = best;
        P.qidx[b * P.nq + i] = best;
    }
    P.qnum[b] = nq;
    P.query_num[b] = nq;
    for (int i = 0; i < P.qout; ++i)
        for (int d = 0; d < 7; ++d)
            P.box_f[((size_t)b * P.qout + i) * 7 + d] =
                (i < nq && d >= 3 && d < 6) ? (float)P.boxes[((size_t)b * P.L + taken[i]) * 7 + d] : 0.f;
    if (P.gt_box_f)
        for (int i = 0; i < P.qout; ++i)
            for (int d = 0; d < 7; ++d)
                P.gt_box_f[((size_t)b * P.qout + i) * 7 + d] =
                    (i < nq && d >= 3 && d < 6) ? P.gt_traj[((size_t)b * P.L + taken[i]) * 7 + d] : 0.f;
}

// ---- select: the k ranks of 0..n-1 with the smallest keys mix64(base + r), sorted, into out; called by a whole 256-thread block ----
__device__ void select_k(unsigned long long base, int n, int k, int* out) {
    if (n <= k) {
        for (int r = threadIdx.x; r < n; r += blockDim.x) out[r] = r;
        return;
    }
    __shared__ unsigned hist[256];
    __shared__ unsigned long long s_prefix, s_mask;
    __shared__ int s_need, s_done, s_warp[8];
    if (threadIdx.x == 0) { s_prefix = 0; s_mask = 0; s_need = k; s_done = 0; }
    // radix select of the k-th smallest key, 8 bits per pass from the top, stopping once its bucket is taken whole
    for (int shift = 56; shift >= 0; shift -= 8) {
        hist[threadIdx.x] = 0;
        __syncthreads();
        const unsigned long long prefix = s_prefix, mask = s_mask;
        for (int r = threadIdx.x; r < n; r += blockDim.x) {
            const unsigned long long key = mix64(base + (unsigned long long)r);
            if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int c = 0, d = 0;
            for (; d < 255; ++d) { if (c + (int)hist[d] >= s_need) break; c += hist[d]; }
            s_need -= c;
            s_prefix |= (unsigned long long)d << shift;
            s_mask |= 255ull << shift;
            s_done = (int)hist[d] == s_need;
        }
        __syncthreads();
        if (s_done) break;
    }
    const unsigned long long thr = s_prefix | ~s_mask;      // exactly k keys are <= thr
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int run = 0;
    for (int r0 = 0; r0 < n; r0 += 256) {                   // ordered compaction: ranks come out sorted
        const int r = r0 + threadIdx.x;
        const bool s = r < n && mix64(base + (unsigned long long)r) <= thr;
        const unsigned bal = __ballot_sync(0xffffffffu, s);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) { const int c = s_warp[w]; before += w < warp ? c : 0; total += c; }
        if (s) out[run + before + __popc(bal & ((1u << lane) - 1u))] = r;
        run += total;
        __syncthreads();
    }
}

// ---- select: one block per selection ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_rd_select(RdParams P) {
    const int id = blockIdx.x;
    int b, slot, stream, n, k;
    int* out;
    if (P.kind == RD_GRM) {
        b = id / (P.nq + 1);
        const int i = id % (P.nq + 1);
        if (i < P.nq) {
            if (i >= P.qnum[b]) return;
            slot = P.qidx[b * P.nq + i]; stream = ST_GRM_Q; k = P.kq; n = P.n[(size_t)b * P.L + slot];
            out = sel_list(P, b, i, ST_GRM_Q);
        } else {
            slot = 0; stream = ST_GRM_M; k = P.km; n = P.gtot[b];
            out = sel_list(P, b, 0, ST_GRM_M);
        }
    } else {
        const int per = P.kind == RD_PRM ? 2 : 1;
        const int t = id / per;
        b = t / P.L; slot = t % P.L;
        if (slot >= track_len(P, b)) return;
        stream = P.kind == RD_CRM ? ST_CRM : (id % per ? ST_PRM_M : ST_PRM_Q);
        k = stream == ST_PRM_M ? P.km : P.kq;
        n = P.n[t];
        out = sel_list(P, b, slot, stream);
    }
    select_k(key_base(P.seed, P.uid[b], slot, stream), n, k, out);
}

// ---- fill: every row no point lands in -----------------------------------------------------------------------------------------
__global__ void k_rd_fill(RdParams P) {
    const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (P.kind == RD_GRM) {
        const long long nq_rows = (long long)P.B * P.qout * P.kq;
        if (id < nq_rows) {
            const int s = id % P.kq, qi = (id / P.kq) % P.qout, b = id / ((long long)P.kq * P.qout);
            const bool pad = qi >= P.qnum[b] || s >= min(P.n[(size_t)b * P.L + P.qidx[b * P.nq + qi]], P.kq);
            if (pad) for (int d = 0; d < 4; ++d) P.q_pts[id * 4 + d] = 0.f;
            return;
        }
        const long long m = id - nq_rows;
        if (m >= (long long)P.B * P.km) return;
        const int s = m % P.km, b = m / P.km;
        if (s >= min(P.gtot[b], P.km)) for (int d = 0; d < 11; ++d) P.m_pts[m * 11 + d] = 0.f;
        return;
    }
    const long long nq_rows = (long long)P.B * P.L * P.kq, nm_rows = P.kind == RD_PRM ? (long long)P.B * P.L * P.km : 0;
    float* o;
    int s, t, k;
    if (id < nq_rows) { k = P.kq; s = id % k; t = id / k; o = P.q_pts + id * P.C; }
    else if (id < nq_rows + nm_rows) { k = P.km; s = (id - nq_rows) % k; t = (id - nq_rows) / k; o = P.m_pts + (id - nq_rows) * P.C; }
    else return;
    const int b = t / P.L, j = t % P.L;
    if (j >= track_len(P, b)) { for (int d = 0; d < P.C; ++d) o[d] = 0.f; return; }
    if (s < min(P.n[t], k)) return;                                        // a point lands here
    const double e[3] = {0.0, 0.0, 0.0};
    emit_p2co(o, e, 0.f, P.bx[t], P.with_class, P.cls[b]);
}

// the RdParams arrays that live in the workspace; n and sel serve when the caller passes no counts / sel
struct RdWs { RdBox* bx; int *cc, *n, *goff, *gtot, *qnum, *qidx, *sel, n_chunks; };

static RdWs carve_rd(DzCarve& cv, int kind, int B, int L, int max_frame_points, int kq, int km, int nq) {
    const size_t T = (size_t)B * L;
    RdWs w;
    w.n_chunks = dz_cdiv(max(max_frame_points, 1), RD_CHUNK);
    w.bx = cv.take<RdBox>(T);
    w.cc = cv.take<int>(T * w.n_chunks); w.n = cv.take<int>(T); w.goff = cv.take<int>(T);
    w.gtot = cv.take<int>(B); w.qnum = cv.take<int>(B); w.qidx = cv.take<int>((size_t)B * nq);
    w.sel = cv.take<int>(kind == RD_PRM ? T * (kq + km) : kind == RD_CRM ? T * kq : (size_t)B * (nq * kq + km));
    return w;
}

// the passes of one build: prep, count, scan, (GRM: per track), select, fill, write
static void launch_rd(const RdParams& P, cudaStream_t st) {
    const int T = P.B * P.L;
    k_rd_prep<<<dz_cdiv(T, 128), 128, 0, st>>>(P);
    dim3 grid(T, P.n_chunks);
    k_rd_crop<0><<<grid, 256, 0, st>>>(P);
    k_rd_scan<<<dz_cdiv(T, 128), 128, 0, st>>>(P);
    if (P.kind == RD_GRM) k_rd_track<<<dz_cdiv(P.B, 64), 64, 0, st>>>(P);
    const int n_sel = P.kind == RD_GRM ? P.B * (P.nq + 1) : T * (P.kind == RD_PRM ? 2 : 1);
    k_rd_select<<<n_sel, 256, 0, st>>>(P);
    const long long rows = P.kind == RD_GRM ? (long long)P.B * (P.qout * P.kq + P.km) : (long long)T * (P.kq + P.km);
    k_rd_fill<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(P);
    k_rd_crop<1><<<grid, 256, 0, st>>>(P);
}

extern "C" size_t dz_refine_inputs_ws_bytes(int kind, int B, int L, int max_frame_points, int kq, int km, int nq) {
    return dz_carve_bytes(carve_rd, kind, B, L, max_frame_points, kq, km, nq);
}

extern "C" int dz_refine_inputs(int kind, const float* points, int pt_stride, const int32_t* frame_offsets, int n_frames,
                                int max_frame_points, const double* poses, const double* boxes, const int32_t* frame_of_box,
                                const float* scores, const int32_t* box_num, const int32_t* cls, const int64_t* track_uid, int B,
                                int L, int kq, int km, int nq, int q_out, int with_class, double enlarge_scale, int crop_on_bev,
                                int crop, unsigned long long seed, float* q_pts, float* m_pts, float* traj, float* box_f,
                                float* track_f, int32_t* query_num, int32_t* counts, int32_t* sel, void* ws, size_t ws_bytes,
                                dz_stream_t stream) {
    DZ_CHECK_ARG(kind >= RD_PRM && kind <= RD_GRM && pt_stride >= 5 && frame_offsets && n_frames >= 1 && max_frame_points >= 0 &&
                 poses && boxes && frame_of_box && scores && box_num && cls && track_uid && B >= 0 && L >= 1 && kq >= 1 &&
                 q_pts && box_f && (points || max_frame_points == 0));
    DZ_CHECK_ARG(kind == RD_CRM || km >= 1);
    DZ_CHECK_ARG(kind != RD_PRM || (m_pts && traj && track_f));
    DZ_CHECK_ARG(kind != RD_GRM || (m_pts && traj && query_num && nq >= 1 && nq <= 8 && q_out >= 0 && q_out <= nq));
    if (B == 0) return DZ_OK;
    DZ_CHECK_WS(dz_refine_inputs_ws_bytes(kind, B, L, max_frame_points, kq, km, nq));
    RdParams P = {};
    P.pts = points; P.pstride = pt_stride; P.foff = frame_offsets; P.F = n_frames;
    P.poses = poses; P.boxes = boxes; P.fob = frame_of_box; P.scores = scores; P.box_num = box_num; P.cls = cls;
    P.uid = (const long long*)track_uid;
    P.B = B; P.L = L; P.kind = kind; P.with_class = with_class ? 1 : 0; P.C = kind == RD_GRM ? 4 : 32 + 3 * P.with_class;
    P.kq = kq; P.km = kind == RD_CRM ? 0 : km; P.nq = nq; P.qout = q_out; P.crop = crop ? 1 : 0; P.bev = crop_on_bev ? 1 : 0;
    P.enlarge = enlarge_scale; P.seed = seed;
    DzCarve cv((char*)ws);
    const RdWs w = carve_rd(cv, kind, B, L, max_frame_points, kq, km, nq);
    P.n_chunks = w.n_chunks; P.bx = w.bx; P.cc = w.cc; P.n = counts ? counts : w.n; P.goff = w.goff;
    P.gtot = w.gtot; P.qnum = w.qnum; P.qidx = w.qidx; P.sel = sel ? sel : w.sel;
    P.q_pts = q_pts; P.m_pts = m_pts; P.traj = traj; P.box_f = box_f; P.track_f = track_f; P.query_num = query_num;
    launch_rd(P, (cudaStream_t)stream);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---- training samples ------------------------------------------------------------------------------------------------------------
// the draw of one track: one block of 256 threads
struct RdDraw {
    const int* box_num; const unsigned char* matched; const long long* uid;
    int B, L, kind, nq; unsigned long long seed;
    int* elig; int* kept; int* n_kept; int* qsel; int* init; unsigned char* flip;
};

__global__ void __launch_bounds__(256) k_rd_draw(RdDraw D) {
    const int b = blockIdx.x;
    const int L = min(max(D.box_num[b], 0), D.L);
    const long long uid = D.uid[b];
    int* elig = D.elig + (size_t)b * D.L;
    int* kept = D.kept + (size_t)b * D.L;
    __shared__ int s_m, s_n;
    if (threadIdx.x == 0) {                                                  // eligible slots, ascending
        int m = 0;
        for (int j = 0; j < L; ++j)
            if (!D.matched || D.matched[(size_t)b * D.L + j]) elig[m++] = j;
        const int lo = min(5, m);
        const int n = m ? lo + (int)(mix64(key_base(D.seed, uid, 0, ST_TR_COUNT)) % (unsigned long long)(m - lo + 1)) : 0;
        s_m = m; s_n = n;
        D.n_kept[b] = n;
        if (D.init) D.init[b] = n ? (int)(mix64(key_base(D.seed, uid, 0, ST_TR_INIT)) % (unsigned long long)n) : 0;
    }
    __syncthreads();
    const int m = s_m, n = s_n;
    select_k(key_base(D.seed, uid, 0, ST_TR_KEEP), m, n, kept);              // ranks among the eligible slots
    __syncthreads();
    for (int i = threadIdx.x; i < D.L; i += blockDim.x) kept[i] = i < n ? elig[kept[i]] : -1;
    if (D.qsel) {
        int* q = D.qsel + (size_t)b * D.nq;
        const int nq = min(D.nq, n);
        select_k(key_base(D.seed, uid, 0, ST_TR_QUERY), n, nq, q);
        __syncthreads();
        for (int i = nq + threadIdx.x; i < D.nq; i += blockDim.x) q[i] = -1;
    }
    if (D.flip) {
        const unsigned long long base = key_base(D.seed, uid, 0, ST_TR_FLIP);
        for (int i = threadIdx.x; i < D.L; i += blockDim.x)
            D.flip[(size_t)b * D.L + i] = i < n ? (unsigned char)(mix64(base + (unsigned long long)i) >> 63) : 0;
    }
}

static int* carve_draw(DzCarve& cv, int B, int L) { return cv.take<int>((size_t)B * L); }

extern "C" size_t dz_refine_train_draw_ws_bytes(int B, int L) { return dz_carve_bytes(carve_draw, B, L); }

extern "C" int dz_refine_train_draw(int kind, const int32_t* box_num, const uint8_t* matched, const int64_t* track_uid, int B, int L,
                                    int nq, unsigned long long seed, long long epoch, int32_t* kept, int32_t* n_kept,
                                    int32_t* query_slots, int32_t* init_slot, uint8_t* flip, void* ws, size_t ws_bytes,
                                    dz_stream_t stream) {
    DZ_CHECK_ARG(kind >= RD_PRM && kind <= RD_GRM && box_num && track_uid && B >= 0 && L >= 1 && kept && n_kept);
    DZ_CHECK_ARG(kind != RD_GRM || (matched && query_slots && flip && nq >= 1 && nq <= 8));
    DZ_CHECK_ARG(kind != RD_PRM || (matched && init_slot));
    DZ_CHECK_ARG(kind != RD_CRM || init_slot);
    if (B == 0) return DZ_OK;
    DZ_CHECK_WS(dz_refine_train_draw_ws_bytes(B, L));
    DzCarve cv((char*)ws);
    RdDraw D;
    D.box_num = box_num; D.matched = kind != RD_CRM ? matched : nullptr; D.uid = (const long long*)track_uid;
    D.B = B; D.L = L; D.kind = kind; D.nq = nq; D.seed = epoch_seed(seed, epoch);
    D.elig = carve_draw(cv, B, L); D.kept = kept; D.n_kept = n_kept;
    D.qsel = kind == RD_GRM ? query_slots : nullptr; D.init = kind != RD_GRM ? init_slot : nullptr;
    D.flip = kind == RD_GRM ? flip : nullptr;
    k_rd_draw<<<B, 256, 0, (cudaStream_t)stream>>>(D);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// the kept slots of each track -> the derived track table (boxes, frame_of_box, scores) and the kept targets: gt_geo_trajectory
// (GRM, f32 world, zero padded), the kept ground truth (PRM, f64 world, zero padded) and iou (CRM, -1 padded).  One thread per
// derived slot.
__global__ void k_rd_gather(const double* __restrict__ boxes, const int* __restrict__ fob, const float* __restrict__ scores,
                            const int* __restrict__ kept, const int* __restrict__ n_kept, const double* __restrict__ gt_boxes,
                            const float* __restrict__ iou, int B, int L, double* __restrict__ dboxes, int* __restrict__ dfob,
                            float* __restrict__ dscores, float* __restrict__ gt_traj, double* __restrict__ dgt,
                            float* __restrict__ iou_out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * L) return;
    const int b = t / L, i = t % L;
    const bool live = i < min(max(n_kept[b], 0), L);
    const size_t s = live ? (size_t)b * L + kept[t] : 0;
    for (int d = 0; d < 7; ++d) dboxes[(size_t)t * 7 + d] = live ? boxes[s * 7 + d] : 0.0;
    dfob[t] = live ? fob[s] : 0;
    dscores[t] = live ? scores[s] : 0.f;
    if (gt_traj) for (int d = 0; d < 7; ++d) gt_traj[(size_t)t * 7 + d] = live ? (float)gt_boxes[s * 7 + d] : 0.f;
    if (dgt) for (int d = 0; d < 7; ++d) dgt[(size_t)t * 7 + d] = live ? gt_boxes[s * 7 + d] : 0.0;
    if (iou_out) iou_out[t] = live ? iou[s] : -1.f;
}

struct RdTrainWs { double* boxes; int* fob; float* scores; double* gt; RdWs rd; };

static RdTrainWs carve_rd_train(DzCarve& cv, int kind, int B, int L, int max_frame_points, int kq, int km, int nq) {
    RdTrainWs w;
    w.boxes = cv.take<double>((size_t)B * L * 7);
    w.fob = cv.take<int>((size_t)B * L);
    w.scores = cv.take<float>((size_t)B * L);
    w.gt = kind == RD_PRM ? cv.take<double>((size_t)B * L * 7) : nullptr;
    w.rd = carve_rd(cv, kind, B, L, max_frame_points, kq, km, nq);
    return w;
}

extern "C" size_t dz_refine_train_inputs_ws_bytes(int kind, int B, int L, int max_frame_points, int kq, int km, int nq) {
    return dz_carve_bytes(carve_rd_train, kind, B, L, max_frame_points, kq, km, nq);
}

// what every training build shares: the gather of the kept slots (with the kind's kept targets) and the RdParams of the passes on
// the derived table; the caller adds the kind's own outputs and launches
static RdParams rd_train_params(const RdTrainWs& w, int kind, const float* points, int pt_stride, const int32_t* frame_offsets,
                                int n_frames, const double* poses, const double* boxes, const int32_t* frame_of_box,
                                const float* scores, const int32_t* cls, const int64_t* track_uid, const double* gt_boxes,
                                const float* iou, int B, int L, int kq, int km, int nq, int q_out, double enlarge_scale,
                                int crop_on_bev, int crop, unsigned long long seed, long long epoch, const int32_t* kept,
                                const int32_t* n_kept, float* gt_traj, float* iou_out, int32_t* counts, int32_t* sel,
                                cudaStream_t st) {
    k_rd_gather<<<dz_cdiv(B * L, 128), 128, 0, st>>>(boxes, frame_of_box, scores, kept, n_kept, gt_boxes, iou, B, L, w.boxes, w.fob,
                                                     w.scores, kind == RD_GRM ? gt_traj : nullptr, w.gt,
                                                     kind == RD_CRM ? iou_out : nullptr);
    RdParams P = {};
    P.pts = points; P.pstride = pt_stride; P.foff = frame_offsets; P.F = n_frames;
    P.poses = poses; P.boxes = w.boxes; P.fob = w.fob; P.scores = w.scores; P.box_num = n_kept; P.cls = cls;
    P.uid = (const long long*)track_uid;
    P.B = B; P.L = L; P.kind = kind; P.with_class = 0; P.C = kind == RD_GRM ? 4 : 32;
    P.kq = kq; P.km = kind == RD_CRM ? 0 : km; P.nq = nq; P.qout = q_out; P.crop = crop ? 1 : 0; P.bev = crop_on_bev ? 1 : 0;
    P.enlarge = enlarge_scale; P.seed = epoch_seed(seed, epoch);
    P.n_chunks = w.rd.n_chunks; P.bx = w.rd.bx; P.cc = w.rd.cc; P.n = counts ? counts : w.rd.n; P.goff = w.rd.goff;
    P.gtot = w.rd.gtot; P.qnum = w.rd.qnum; P.qidx = w.rd.qidx; P.sel = sel ? sel : w.rd.sel;
    return P;
}

extern "C" int dz_refine_train_inputs(int kind, const float* points, int pt_stride, const int32_t* frame_offsets, int n_frames,
                                      int max_frame_points, const double* poses, const double* boxes, const int32_t* frame_of_box,
                                      const float* scores, const int32_t* cls, const int64_t* track_uid, const double* gt_boxes,
                                      const float* iou, int B, int L, int kq, int km, int nq, int q_out, double enlarge_scale,
                                      int crop_on_bev, int crop, unsigned long long seed, long long epoch, const int32_t* kept,
                                      const int32_t* n_kept, const int32_t* query_slots, const int32_t* init_slot,
                                      const uint8_t* flip, float* q_pts, float* m_pts, float* traj, float* box_f, float* gt_box_f,
                                      float* gt_traj, float* iou_out, int32_t* query_num, int32_t* counts, int32_t* sel, void* ws,
                                      size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG((kind == RD_CRM || kind == RD_GRM) && pt_stride >= 5 && frame_offsets && n_frames >= 1 && max_frame_points >= 0 &&
                 poses && boxes && frame_of_box && scores && cls && track_uid && B >= 0 && L >= 1 && kq >= 1 && kept && n_kept &&
                 q_pts && box_f && (points || max_frame_points == 0));
    DZ_CHECK_ARG(kind != RD_GRM || (gt_boxes && query_slots && m_pts && traj && gt_box_f && gt_traj && query_num && km >= 1 &&
                                    nq >= 1 && nq <= 8 && q_out >= 0 && q_out <= nq));
    DZ_CHECK_ARG(kind != RD_CRM || (iou && init_slot && iou_out));
    if (B == 0) return DZ_OK;
    DZ_CHECK_WS(dz_refine_train_inputs_ws_bytes(kind, B, L, max_frame_points, kq, km, nq));
    DzCarve cv((char*)ws);
    const RdTrainWs w = carve_rd_train(cv, kind, B, L, max_frame_points, kq, km, nq);
    cudaStream_t st = (cudaStream_t)stream;
    RdParams P = rd_train_params(w, kind, points, pt_stride, frame_offsets, n_frames, poses, boxes, frame_of_box, scores, cls,
                                 track_uid, gt_boxes, iou, B, L, kq, km, nq, q_out, enlarge_scale, crop_on_bev, crop, seed, epoch,
                                 kept, n_kept, gt_traj, iou_out, counts, sel, st);
    P.q_pts = q_pts; P.m_pts = m_pts; P.traj = kind == RD_GRM ? traj : nullptr; P.box_f = box_f; P.query_num = query_num;
    if (kind == RD_GRM) { P.qsel = query_slots; P.flip = flip; P.gt_traj = gt_traj; P.gt_box_f = gt_box_f; }
    else P.init = init_slot;
    launch_rd(P, st);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

extern "C" size_t dz_position_train_inputs_ws_bytes(int B, int L, int max_frame_points, int kq, int km) {
    return dz_carve_bytes(carve_rd_train, (int)RD_PRM, B, L, max_frame_points, kq, km, 1);
}

extern "C" int dz_position_train_inputs(const float* points, int pt_stride, const int32_t* frame_offsets, int n_frames,
                                        int max_frame_points, const double* poses, const double* boxes, const int32_t* frame_of_box,
                                        const float* scores, const int32_t* cls, const int64_t* track_uid, const double* gt_boxes,
                                        int B, int L, int kq, int km, double enlarge_scale, int crop_on_bev, int crop,
                                        unsigned long long seed, long long epoch, const int32_t* kept, const int32_t* n_kept,
                                        const int32_t* init_slot, float* q_pts, float* m_pts, float* traj, float* gt_traj,
                                        float* padding_mask, float* init_box, int32_t* counts, int32_t* sel, void* ws,
                                        size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(pt_stride >= 5 && frame_offsets && n_frames >= 1 && max_frame_points >= 0 && poses && boxes && frame_of_box &&
                 scores && cls && track_uid && gt_boxes && B >= 0 && L >= 1 && kq >= 1 && km >= 1 && kept && n_kept && init_slot &&
                 q_pts && m_pts && traj && gt_traj && padding_mask && init_box && (points || max_frame_points == 0));
    if (B == 0) return DZ_OK;
    DZ_CHECK_WS(dz_position_train_inputs_ws_bytes(B, L, max_frame_points, kq, km));
    DzCarve cv((char*)ws);
    const RdTrainWs w = carve_rd_train(cv, RD_PRM, B, L, max_frame_points, kq, km, 1);
    cudaStream_t st = (cudaStream_t)stream;
    RdParams P = rd_train_params(w, RD_PRM, points, pt_stride, frame_offsets, n_frames, poses, boxes, frame_of_box, scores, cls,
                                 track_uid, gt_boxes, nullptr, B, L, kq, km, 1, 0, enlarge_scale, crop_on_bev, crop, seed, epoch,
                                 kept, n_kept, nullptr, nullptr, counts, sel, st);
    P.q_pts = q_pts; P.m_pts = m_pts; P.traj = traj; P.box_f = padding_mask; P.track_f = init_box;
    P.init = init_slot; P.gt_w = w.gt; P.gt_pos = gt_traj;
    launch_rd(P, st);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---- crop once: every in-box point row of every box slot, copied to rows[rbase[t] + rank] --------------------------------------
static RdWs carve_crop(DzCarve& cv, int B, int L, int max_frame_points) {
    const size_t T = (size_t)B * L;
    RdWs w = {};
    w.n_chunks = dz_cdiv(max(max_frame_points, 1), RD_CHUNK);
    w.bx = cv.take<RdBox>(T);
    w.cc = cv.take<int>(T * w.n_chunks);
    return w;
}

extern "C" size_t dz_crop_tracks_ws_bytes(int B, int L, int max_frame_points) {
    return dz_carve_bytes(carve_crop, B, L, max_frame_points);
}

extern "C" int dz_crop_tracks(const float* points, int pt_stride, int width, const int32_t* frame_offsets, int n_frames,
                              int max_frame_points, const double* poses, const double* boxes, const int32_t* frame_of_box,
                              const int32_t* box_num, int B, int L, double enlarge_scale, int crop_on_bev, int32_t* counts,
                              const int32_t* row_base, float* rows, void* ws, size_t ws_bytes, dz_stream_t stream) {
    DZ_CHECK_ARG(pt_stride >= 5 && width >= 5 && width <= pt_stride && frame_offsets && n_frames >= 1 && max_frame_points >= 0 &&
                 poses && boxes && frame_of_box && box_num && B >= 0 && L >= 1 && counts && (points || max_frame_points == 0) &&
                 (!rows == !row_base));
    if (B == 0) return DZ_OK;
    DZ_CHECK_WS(dz_crop_tracks_ws_bytes(B, L, max_frame_points));
    DzCarve cv((char*)ws);
    const RdWs w = carve_crop(cv, B, L, max_frame_points);
    RdParams P = {};
    P.pts = points; P.pstride = pt_stride; P.foff = frame_offsets; P.F = n_frames;
    P.poses = poses; P.boxes = boxes; P.fob = frame_of_box; P.box_num = box_num;
    P.B = B; P.L = L; P.kind = RD_CROP; P.C = width; P.crop = 1; P.bev = crop_on_bev ? 1 : 0; P.enlarge = enlarge_scale;
    P.n_chunks = w.n_chunks; P.bx = w.bx; P.cc = w.cc; P.n = counts; P.rbase = row_base; P.rows = rows;
    cudaStream_t st = (cudaStream_t)stream;
    const int T = B * L;
    dim3 grid(T, P.n_chunks);
    k_rd_prep<<<dz_cdiv(T, 128), 128, 0, st>>>(P);
    k_rd_crop<0><<<grid, 256, 0, st>>>(P);
    k_rd_scan<<<dz_cdiv(T, 128), 128, 0, st>>>(P);
    if (rows) k_rd_crop<1><<<grid, 256, 0, st>>>(P);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

// ---- revert_to_each_frame: one thread per box slot --------------------------------------------------------------------------------
// PRM (kind 0): pred (B, L, 7) in the init-box frame -> world (box_coords_transform) -> lidar (world_to_lidar).
// GRM (kind 2): pred (B, 7); its size written into each world box -> lidar.  Rows past box_num are zero.
__global__ void k_rd_revert(int kind, const float* __restrict__ pred, const double* __restrict__ poses, int F,
                            const double* __restrict__ boxes, const int* __restrict__ fob, const int* __restrict__ box_num, int B, int L,
                            double* __restrict__ lidar, double* __restrict__ world) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * L) return;
    const int b = t / L, j = t % L, n = min(max(box_num[b], 0), L);
    double w[7], l[7];
    if (j >= n) {
        for (int d = 0; d < 7; ++d) lidar[(size_t)t * 7 + d] = world[(size_t)t * 7 + d] = 0.0;
        return;
    }
    if (kind == RD_PRM) {
        const double* bi = boxes + ((size_t)b * L + n / 2) * 7;
        const double yi = wrap_pi(bi[6]), c = cos(yi), s = sin(yi);
        const float* p = pred + (size_t)t * 7;
        w[0] = c * p[0] - s * p[1] + bi[0];
        w[1] = s * p[0] + c * p[1] + bi[1];
        w[2] = (double)p[2] + bi[2];
        for (int d = 3; d < 6; ++d) w[d] = p[d];
        w[6] = wrap_pi((double)p[6] + yi);
    } else {
        for (int d = 0; d < 7; ++d) w[d] = boxes[(size_t)t * 7 + d];
        for (int d = 3; d < 6; ++d) w[d] = pred[(size_t)b * 7 + d];
    }
    const double* P = poses + (size_t)min(max(fob[t], 0), F - 1) * 16;
    // inverse of the rigid pose: R^T, -R^T t
    for (int r = 0; r < 3; ++r)
        l[r] = P[0 * 4 + r] * (w[0] - P[3]) + P[1 * 4 + r] * (w[1] - P[7]) + P[2 * 4 + r] * (w[2] - P[11]);
    for (int d = 3; d < 6; ++d) l[d] = w[d];
    l[6] = w[6] + atan2(P[0 * 4 + 1], P[0 * 4 + 0]);
    for (int d = 0; d < 7; ++d) { lidar[(size_t)t * 7 + d] = l[d]; world[(size_t)t * 7 + d] = w[d]; }
}

extern "C" int dz_refine_revert(int kind, const float* pred, const double* poses, int n_frames, const double* boxes,
                                const int32_t* frame_of_box, const int32_t* box_num, int B, int L, double* lidar, double* world,
                                dz_stream_t stream) {
    DZ_CHECK_ARG((kind == RD_PRM || kind == RD_GRM) && pred && poses && n_frames >= 1 && boxes && frame_of_box && box_num &&
                 B >= 0 && L >= 1 && lidar && world);
    if (B == 0) return DZ_OK;
    k_rd_revert<<<dz_cdiv(B * L, 128), 128, 0, (cudaStream_t)stream>>>(kind, pred, poses, n_frames, boxes, frame_of_box, box_num, B,
                                                                         L, lidar, world);
    DZ_LAUNCH_CHECK();
    return DZ_OK;
}

/*
 * detzero_b200.h -- C ABI of libdetzero_b200.so (sm_90a).
 *
 * The reference (PJLab-ADG/DetZero) has no C ABI: its native ops are pybind11 modules taking at::Tensor
 * (utils/detzero_utils/ops/iou3d_nms/src/iou3d_nms_api.cpp:10-17) and its sparse-conv / voxelizer arithmetic
 * lives in the third-party spconv wheel.  Each entry point below names the reference interface it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless marked "host"; the caller owns all buffers incl. workspace
 *   - functions only enqueue work on `stream` (a cudaStream_t): no malloc, no sync, no host loop
 *   - element counts that are only known on the device are passed as `const int* d_n` (device scalar) together
 *     with a host-side capacity `cap`; kernels are persistent / grid-stride over `cap` and read `*d_n`
 *   - return 0 on success, <0 on error (never exit(); contrast iou3d_nms.cpp:14-26); dz_last_error_string()
 *   - feature tensors are row-major (rows, channels); dense maps are NHWC
 *
 * Grid index ("coordinate index"): for a lattice (B, D, H, W) a bitmap of occupied cells + an exclusive
 * popcount prefix per 32-bit word (+ optional permutation rank->row).  cell = b*cells_pad + (z*H+y)*W+x with
 * cells_pad = round_up(D*H*W, 32).  Rank order == ascending (b,z,y,x).
 */
#ifndef DETZERO_B200_H
#define DETZERO_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef void* dz_stream_t;           /* cudaStream_t */

enum { DZ_OK = 0, DZ_ERR_ARG = -1, DZ_ERR_CUDA = -2, DZ_ERR_WORKSPACE = -3, DZ_ERR_UNSUPPORTED = -4 };
enum { DZ_F32 = 0, DZ_TF32 = 1, DZ_BF16 = 2, DZ_TF32X3 = 3, DZ_BF16X2 = 4 };   /* arithmetic mode of GEMM-shaped kernels:
   F32 = fp32 FMA; TF32 = one wgmma TF32 pass; TF32X3 = hi/lo split, 3 TF32 passes, fp32-level accuracy (sparse conv);
   BF16 / BF16X2 = bf16 operand planes (1 plane: bf16 storage; 2 planes: x = p0 + p1, 16 significand bits in 4 bytes,
   fp32-level accuracy at the cost of one TF32 pass), sparse conv only: dz_spconv_fwd_planes */

int         dz_version(void);
int         dz_sm_arch(void);                      /* 90 : built for sm_90a */
const char* dz_last_error_string(void);            /* host string, thread-local */

/* ---- grid index ---------------------------------------------------------------------------------------- */
size_t dz_grid_index_words(int B, int D, int H, int W);          /* number of u32 words in bitmap == prefix */
size_t dz_scan_ws_bytes(size_t n_words);
/* prefix[w] = base + popcount(bitmap[0..w)), *d_total = base + popcount(all); base = d_base ? *d_base : 0 */
int dz_grid_index_scan(const uint32_t* bitmap, uint32_t* prefix, size_t n_words, const int* d_base,
                       int* d_total, void* ws, size_t ws_bytes, dz_stream_t stream);
/* arbitrary site list -> index (+perm: rank -> row).  Replaces the hash table spconv builds inside
 * SparseConvTensor/indice_dict (backbone3d.py:190-195).  bitmap must be zero on entry. */
int dz_grid_index_from_coords(const int32_t* coords, const int* d_n, int cap, int B, int D, int H, int W,
                              uint32_t* bitmap, uint32_t* prefix, int32_t* perm, int* d_total,
                              void* ws, size_t ws_bytes, dz_stream_t stream);

/* ---- voxelization -------------------------------------------------------------------------------------- */
/* Hard voxelization of ONE cloud, order-exact with spconv.utils.Point2VoxelCPU3d.point_to_voxel as driven by
 * detection/detzero_det/datasets/processor/data_processor.py:61-91 (first-appearance voxel ids, first max_pts
 * points kept in input order, voxel cap in appearance order), fused with MeanVFE.forward (vfe.py:66-83).
 *   points (n, point_stride) f32; the c feature columns [xyz_off, xyz_off+c) start with x,y,z and are copied
 *   verbatim (xyz_off = 1 for a collated (N,1+C) [b,x,y,z,..] tensor, 0 for a raw (N,C) cloud)
 *   voxels (cap, max_pts, c) ; coords (cap,4) [batch_idx,z,y,x] ; num_per_voxel (cap) ; mean (cap,c) or NULL
 *   d_counters[0] = rows already used in voxels/coords (in/out), d_counters[1] = ranks already used in the
 *   index (in/out), d_counters[2] = rows wanted (in/out; > [0] iff `cap` was too small): calling once per frame with batch_idx = 0..B-1 on one stream builds a collated batch
 *   (dataset.py:260-303) without a host sync.
 *   index_* : level-0 grid index over lattice (B, iD, iH, iW) (iD = sparse_shape z = grid z + 1,
 *   backbone3d.py:133); bitmap must be zero before the first frame of a batch. */
size_t dz_voxelize_hard_ws_bytes(int n_points, int max_pts, int max_voxels, int iD, int iH, int iW);
int dz_voxelize_hard(const float* points, int n, int point_stride, int xyz_off, int c,
                     const float* range_xyz6_host, const float* vsize_xyz3_host, const int* grid_zyx3_host,
                     int max_pts, int max_voxels, int batch_idx,
                     float* voxels, int32_t* coords, int32_t* num_per_voxel, float* mean, int cap,
                     int* d_counters,
                     int B, int iD, int iH, int iW, uint32_t* index_bitmap, uint32_t* index_prefix,
                     int32_t* index_perm,
                     void* ws, size_t ws_bytes, dz_stream_t stream);
/* The same for the B frames of a batch in ONE call (frames = batch indices 0..B-1, d_counters zero or carried on entry):
 * the frames run on internal streams forked from / joined to `stream` and only wait for each other's running totals, so
 * their latency-bound kernels overlap.  points_host / n_host are HOST arrays of device pointers / point counts.
 * Identical results to B calls of dz_voxelize_hard in frame order. */
size_t dz_voxelize_hard_batch_ws_bytes(int n_max, int B, int max_pts, int max_voxels, int iD, int iH, int iW);
int dz_voxelize_hard_batch(const float* const* points_host, const int* n_host, int B, int point_stride, int xyz_off, int c,
                           const float* range6_host, const float* vsize3_host, const int* grid_zyx3_host, int max_pts,
                           int max_voxels, float* voxels, int32_t* coords, int32_t* num_per_voxel, float* mean, int cap,
                           int* d_counters, int iD, int iH, int iW, uint32_t* index_bitmap, uint32_t* index_prefix,
                           int32_t* index_perm, void* ws, size_t ws_bytes, dz_stream_t stream);

/* MeanVFE.forward (vfe.py:66-83) on an already voxelized batch: out (M,C) = voxels.sum(1) / max(num,1) */
int dz_mean_vfe(const float* voxels, const int32_t* num_per_voxel, int M, int P, int C, float* out,
                dz_stream_t stream);

/* Dynamic mean voxelization of a collated batch: DynamicMeanVFE.forward (vfe.py:110-147): floor((p-lo)/vs),
 * in-range mask, key b*XYZ + x*YZ + y*Z + z, unique (sorted), scatter_mean of all c columns.
 *   points (n, 1+c) [b,x,y,z,...] ; out feats (cap,c), coords (cap,4) [b,z,y,x] ordered by ascending key ;
 *   *d_m = number of voxels (voxels of rank >= cap are not written).  Each mean is one fp32 sum in ascending point
 *   index followed by an IEEE divide by the count: deterministic, and bit-equal to a sequential scatter on the CPU. */
size_t dz_voxelize_dynamic_ws_bytes(int n_points, int cap, int B, int X, int Y, int Z);
int dz_voxelize_dynamic_mean(const float* points, int n, int c, int B,
                             const float* range_xyz6_host, const float* vsize_xyz3_host,
                             const int* grid_xyz3_host, float* feats, int32_t* coords, int cap, int* d_m,
                             void* ws, size_t ws_bytes, dz_stream_t stream);

/* ---- rulebook ------------------------------------------------------------------------------------------ */
/* Neighbour-table form of the spconv rulebook.  Two layouts, each optional (NULL = not wanted, at least one given):
 *   nbr  k-major  (K, cap):  nbr[k*cap + o] = input row feeding output row o through kernel offset
 *                            k = (kz*KH+ky)*KW+kx, or -1            (exact-fp32 kernel; what the parity tests read)
 *   tab  row-major (cap, 32): tab[o*32 + k] = the same entry for k < K, -1 up to 26, [27] = bit mask of the live
 *                            offsets, [28..31] = 0: one 128-byte line per output row   (tensor-core kernels)
 * The pair set {(k, nbr, o)} equals spconv's indice pairs (SubMConv3d: backbone3d.py:68,93-100,136 ;
 * SparseConv3d: :70-71,169-170,183-184).
 * sched_ws (optional, needs tab; dz_rulebook_schedule_ws_bytes(cap) bytes): the kernel also leaves what
 * dz_rulebook_schedule needs (mask digests, scanned histogram) there. */
int dz_rulebook_subm(const int32_t* coords, const int* d_n, int cap, int B, int D, int H, int W,
                     const int* ksize3_host, const uint32_t* bitmap, const uint32_t* prefix,
                     const int32_t* perm, int32_t* nbr, int32_t* tab, void* sched_ws, dz_stream_t stream);
/* Strided conv: generates the output site set (sorted ascending (b,z,y,x)), its grid index and the table(s).
 * out_bitmap must be zero on entry. */
int dz_rulebook_conv(const int32_t* in_coords, const int* d_n_in, int in_cap, int B,
                     const int* in_dhw3_host, const int* ksize3_host, const int* stride3_host,
                     const int* pad3_host, const uint32_t* in_bitmap, const uint32_t* in_prefix,
                     const int32_t* in_perm, int32_t* out_coords, int* d_n_out, int out_cap,
                     uint32_t* out_bitmap, uint32_t* out_prefix, int32_t* nbr, int32_t* tab,
                     void* ws, size_t ws_bytes, void* sched_ws, dz_stream_t stream);
/* Tile schedule for the tensor-core conv (no reference counterpart; spconv's implicit-GEMM "mask sort" plays the same
 * role).  order (cap + ceil(cap/128) ints): order[p] = output row at tile position p -- rows with alike neighbour
 * masks become adjacent, so a 128-row tile skips the kernel offsets none of its rows uses -- and order[cap + j] = the
 * tile the j-th CTA takes (most live offsets first, capacity tiles beyond the count last).  Hand it to dz_spconv_fwd as
 * row_order; results are bit-identical to the unscheduled call.  sched_ws must be the one the rulebook call filled for this tab. */
size_t dz_rulebook_schedule_ws_bytes(int cap);
int dz_rulebook_schedule(const int32_t* tab, int cap, const int* d_n, int32_t* order, void* sched_ws,
                         size_t ws_bytes, int K, int32_t* tab_tiles, dz_stream_t stream);
/* tab_tiles (optional; ceil(cap/128) * (K+1) * 128 ints): the scheduled table again, TILE-major: tile j = (K+1) planes of 128
 * ints, plane k < K = neighbour row of tile position p through offset k, plane K = the output row order[j*128+p] (-1 beyond the
 * count).  With it `order` must have cap + 2*ceil(cap/128) ints: order[cap + tiles + j] = OR of tile j's row masks.  The
 * persistent bf16-plane conv (dz_spconv_fwd_planes) fetches a tile's block with ONE bulk copy. */

/* ---- sparse convolution -------------------------------------------------------------------------------- */
/* out[o,:] = act( (sum_k in[nbr[k][o],:] @ W[k]) * scale + shift (+ residual[o,:]) )
 * Replaces SubMConv3d/SparseConv3d forward + BatchNorm1d(eval) + bias + residual add + ReLU
 * (backbone3d.py:64-83,105-121).  weight packed (K, cin, cout) f32 (host side repacks spconv's
 * (cout,KD,KH,KW,cin) layout, SURVEY A.3; DZ_TF32 expects (cout, K*cin_pad), DZ_TF32X3 (2, cout, K*cin_pad) = [W_hi ; W_lo]
 * with W_hi = RN_tf32(W), W_lo = RN_tf32(W - W_hi)).  in_rows = allocated rows of `in` (unused).  mode: DZ_F32 exact-fp32 FMA
 * (nbr = k-major table), DZ_TF32 / DZ_TF32X3 one TF32 pass / hi-lo split on the wgmma tensor cores, csrc/spconv_tc.cu
 * (nbr = ROW-major table `tab`, nbr_cap = its rows).
 * row_order: NULL, or the tile schedule of dz_rulebook_schedule (tensor-core modes only). */
int dz_spconv_fwd(const float* in, int cin, int in_rows, const int32_t* nbr, int K, int nbr_cap,
                  const int32_t* row_order, const int* d_n_out,
                  int out_cap, const float* weight, const float* scale, const float* shift,
                  const float* residual, int relu, float* out, int cout, int mode, dz_stream_t stream);
/* out[r, :] = RN_tf32(x[r, :]) (round to nearest, ties to even, 10 explicit mantissa bits) for r < min(*d_n, cap); rows beyond
 * are left alone.  DZ_TF32 reads its input operand by truncation, so an fp32 tensor that enters a DZ_TF32 layer without having
 * come out of one (whose epilogue rounds) is rounded once with this first.  in == out is allowed. */
int dz_round_tf32(const float* x, const int* d_n, int cap, int c, float* out, dz_stream_t stream);

/* Backward of dz_spconv_fwd on the same k-major table (exact fp32; SURVEY.md 8f row 1; the reference trains through spconv's
 * autograd, detection/tools/train_utils.py:59-68).  dz_rulebook_transpose: nbrT (K, cap_in), nbrT[k][j] = o for every pair
 * (k, j = nbr[k][o], o), -1 elsewhere.  dgrad = dz_spconv_fwd(d_out, nbrT, weight^T (K, cout, cin)); the transposed table with its own
 * weights is SparseInverseConv3d (backbone3d.py:72-73).  dz_spconv_wgrad: dW (K, cin, cout) = sum_o in[nbr[k][o]]^T (x) d_out[o]. */
int dz_rulebook_transpose(const int32_t* nbr, int K, int cap_out, const int* d_n_out, int32_t* nbrT, int cap_in,
                          dz_stream_t stream);
int dz_spconv_wgrad(const float* in, int cin, const int32_t* nbr, int K, int nbr_cap, const int* d_n_out, int out_cap,
                    const float* dout, int cout, float* dW, dz_stream_t stream);

/* The same layer on bf16 operand PLANES (modes DZ_BF16: planes = 1, DZ_BF16X2: planes = 2), csrc/spconv_bf16.cu: a persistent
 * warp-specialised wgmma kernel.  Feature tensors `in`, `residual`, `out` are (rows, planes * C) bf16, a row = [p0 | p1] with
 * x ~ p0 (+ p1), p0 = RN_bf16(x), p1 = RN_bf16(x - p0); cin <= 8 is stored padded to 8 channels per plane.  weight: (planes * cout,
 * K * cin_pad) bf16, rows [w0 ; w1] split the same way.  tab = ROW-major table, row_order = NULL or the tile schedule,
 * tab_tiles = NULL or the tile-major table dz_rulebook_schedule wrote next to row_order (fast path).
 * No reference counterpart for the storage format (spconv keeps fp32 rows); dz_to_planes / dz_from_planes convert at the
 * boundary: out[r, p, 0..c_pad) <- x[r, 0..c) (zero padded), x[r, c] <- p0 + p1. */
int dz_spconv_fwd_planes(const void* in, int cin, int in_rows, const int32_t* tab, int K, int tab_rows,
                         const int32_t* row_order, const int* d_n_out, int out_cap, const void* weight,
                         const float* scale, const float* shift, const void* residual, int relu, void* out, int cout,
                         int planes, const int32_t* tab_tiles, dz_stream_t stream);
int dz_to_planes(const float* x, const int* d_n, int cap, int c, int c_pad, int planes, void* out, dz_stream_t stream);
int dz_from_planes(const void* x, const int* d_n, int cap, int c, int planes, float* out, dz_stream_t stream);

/* ---- BEV ------------------------------------------------------------------------------------------------ */
/* SparseConvTensor.dense() + reshape(N, C*D, H, W) (height_compression.py:20-25) into NHWC:
 * out[b,y,x,c*D+z] = feats[i,c].  out must be zero on entry. */
int dz_sparse_to_bev(const float* feats, const int32_t* coords, const int* d_n, int cap, int c,
                     int B, int D, int H, int W, float* out, dz_stream_t stream);
/* the same from a bf16 planes tensor (rows, planes * c) */
int dz_sparse_to_bev_planes(const void* feats, const int32_t* coords, const int* d_n, int cap, int c, int planes,
                            int B, int D, int H, int W, float* out, dz_stream_t stream);
/* NHWC conv2d (cross-correlation) with fused per-channel affine (folded BatchNorm2d / bias) and ReLU; output
 * written at channel offset into a tensor with out_cstride channels (fused torch.cat, backbone2d.py:107-108).
 * weight packed (KH, KW, cin, cout).  Replaces nn.Conv2d(+ZeroPad2d)+BatchNorm2d+ReLU stacks at
 * backbone2d.py:34-48 and center_head.py:25-31,81-88.  in must be 16-byte and out 8-byte aligned (DZ_ERR_ARG otherwise),
 * here and in dz_deconv2d_fwd. */
int dz_conv2d_fwd(const float* in, int B, int H, int W, int cin, int in_cstride, const float* weight, int KH, int KW,
                  int stride, int pad, const float* scale, const float* shift, int relu,
                  float* out, int Ho, int Wo, int cout, int out_coff, int out_cstride, int mode,
                  dz_stream_t stream);
/* ConvTranspose2d with kernel == stride (backbone2d.py:52-60): out[b,y*s+dy,x*s+dx,co] = sum_ci in*W[dy,dx,ci,co]
 * weight packed (s, s, cin, cout). */
int dz_deconv2d_fwd(const float* in, int B, int H, int W, int cin, const float* weight, int s,
                    const float* scale, const float* shift, int relu, float* out, int cout, int out_coff,
                    int out_cstride, int mode, dz_stream_t stream);

/* ---- CenterHead decode + NMS --------------------------------------------------------------------------- */
/* centernet_utils.decode_bbox_from_heatmap / _topk (centernet_utils.py:138-230) on the fused head map
 * (B,H,W,ch) NHWC with channel layout given by ch_* offsets.  Produces, per frame, up to K candidates in
 * descending score order that pass POST_CENTER_LIMIT_RANGE and SCORE_THRESH:
 *   cand_boxes (B,K,7), cand_scores (B,K), cand_labels (B,K) int32 (0-based class), d_cand_n (B). */
size_t dz_centerhead_decode_ws_bytes(int B, int H, int W, int num_class, int K);
int dz_centerhead_decode(const float* head, int B, int H, int W, int ch, int ch_center, int ch_z, int ch_dim,
                         int ch_rot, int ch_iou, int ch_hm, int num_class, int K,
                         const float* range_xyz6_host, const float* vsize_xyz3_host, int fmap_stride,
                         const float* post_limit6_host, float score_thresh, int use_iou,
                         float* cand_boxes, float* cand_scores, int32_t* cand_labels, int* d_cand_n,
                         void* ws, size_t ws_bytes, dz_stream_t stream);
/* Rotated-BEV NMS fully on device: replaces model_nms_utils.class_agnostic_nms -> nms_gpu
 * (model_nms_utils.py:6-25, iou3d_nms_utils.py:154-170, iou3d_nms.cpp:114-160, iou3d_nms_kernel.cu:386-430).
 * Input per frame: n<=cap boxes in descending score order.  Output: out (B, post_max, 9) rows
 * [x,y,z,dx,dy,dz,heading,score,label+label_offset], zero padded, d_out_n (B). */
size_t dz_nms_bev_ws_bytes(int B, int cap);
int dz_nms_bev(const float* boxes, const float* scores, const int32_t* labels, const int* d_n, int B, int cap,
               float thresh, int post_max, int label_offset, float* out, int* d_out_n,
               void* ws, size_t ws_bytes, dz_stream_t stream);
/* pairwise rotated BEV IoU (iou3d_nms_kernel.cu:370-384 boxes_iou_bev_kernel) */
int dz_boxes_iou_bev(const float* boxes_a, int na, const float* boxes_b, int nb, float* out, dz_stream_t stream);

/* ---- on-disk frame -> collated device points (SURVEY.md 8f row 4) ---------------------------------------- */
/* raw: a frame file as waymo_utils.py:284-302 writes it, (n, 6) f32 [x,y,z,intensity,elongation,NLZ_flag], already on the device
 * (pinned-host -> device copy of the file bytes).  Does DatasetTemplate.merge_sweeps (dataset.py:167-196) + the collate batch
 * column (:275-283) on the device: keep NLZ_flag == -1 in file order, tanh(intensity), xyz <- [x y z 1] @ T[:3,:].T in double
 * (transform12_host: row-major 3x4 of inv(current_pose) @ sweep_pose, NULL = identity), append time_offset (with_time),
 * prepend batch_idx.  Rows (1 + 5 + with_time floats) are appended at d_count[0]; d_count[1] = rows wanted (> cap: overflow). */
size_t dz_prepare_points_ws_bytes(int n);
int dz_prepare_points(const float* raw, int n, const double* transform12_host, float time_offset, int with_time, int batch_idx,
                      float* out, int cap, int* d_count, void* ws, size_t ws_bytes, dz_stream_t stream);

/* ---- tracker association matrices + object crop (SURVEY.md 8f rows 2, 3) ---------------------------------- */
/* out (na, nb) = kind(boxes_a[i], boxes_b[j]); boxes are rows of >= 7 floats [x,y,z,dx,dy,dz,heading,...] with row strides
 * lda / ldb floats, so the matrices can be computed straight from the all-gathered (F, 500, 9) detection tensor.
 * kind 0: rotated-BEV IoU (IoUBEV_dis_mat -> boxes_iou_bev_gpu), 1: BEV overlap area (bev_overlap_gpu, the tracker's overlap
 * filter), 2: 3-D IoU (IoU3D_dis_mat -> boxes_iou3d_gpu, iou3d_nms_utils.py:74-107), 3: axis-aligned 2-D IoU on (x,y,dx,dy)
 * (IoU2D_dis_mat).  Replaces tracking/detzero_track/models/tracking_modules/data_association/distance.py:44-141. */
int dz_boxes_pairwise(const float* boxes_a, int na, int lda, const float* boxes_b, int nb, int ldb, int kind, float* out,
                      dz_stream_t stream);
/* Object crop: which points (rows of pt_stride >= 3 floats, x,y,z first) lie inside which box -- points_in_boxes_gpu_v2
 * (roiaware_pool3d_kernel.cu:23-36,352-372; daemon/prepare_object_data.py:264-311) -- as the ORDERED index list the daemon builds
 * on the host: idx (n_boxes, cap) = indices of box t's points in input order (-1 padded, first cap kept), num (n_boxes) = true
 * counts.  dz_points_in_boxes_mask writes the reference's own (n_boxes, n_pts) int32 mask. */
size_t dz_crop_points_ws_bytes(int n_pts, int n_boxes);
int dz_crop_points_in_boxes(const float* points, int n_pts, int pt_stride, const float* boxes, int n_boxes, int ldb,
                            int32_t* idx, int cap, int* num, void* ws, size_t ws_bytes, dz_stream_t stream);
int dz_points_in_boxes_mask(const float* points, int n_pts, int pt_stride, const float* boxes, int n_boxes, int ldb,
                            int32_t* mask, dz_stream_t stream);

/* ---- the DetZero tracker (csrc/tracker.cu) ------------------------------------------------------------------------------ */
/* S sequences of the gathered detection form: boxes (S, F, K, 9) float32 lidar rows [x, y, z, dx, dy, dz, heading, score,
 * label 1..3], counts (S, F), num_frames (S), poses (S, F, 4, 4) float64 lidar -> world.  K <= 512.
 * params (23 doubles): overlap-filter thresholds [3], first-stage IoU [3], second-stage IoU [3], merge [3], score [3] (per class
 * Vehicle, Pedestrian, Cyclist), P[2], Q[2], R, DELTA_T, LEAST_AGE, HEADER_LENGTH.
 * Outputs per sequence s: trk (S, max_tracks, 6) int32 rows [track id, class, first frame, entry count, dynamic, entry offset] of the
 * n_tracks[s] post-processed tracks in id order; ent_box (S, max_entries, 9) float64 world boxes, ent_score, ent_hit (0 / 1 / 2),
 * ent_frame of each entry; kept (S, F, K) u8 the overlap filter's keep flags; overflow[s] != 0 when a capacity was exceeded (the
 * sequence's outputs are then invalid).  One block per sequence, no host synchronisation. */
size_t dz_track_sequences_ws_bytes(int S, int F, int K, int max_tracks, int max_entries);
int dz_track_sequences(const float* boxes, const int* counts, const int* num_frames, const double* poses, int S, int F, int K,
                       const double* params, int max_tracks, int max_entries, int* trk, int* n_tracks, double* ent_box,
                       float* ent_score, int* ent_hit, int* ent_frame, unsigned char* kept, int* overflow, void* ws,
                       size_t ws_bytes, dz_stream_t stream);

/* ---- tracks against ground truth (csrc/track_gt.cu) ------------------------------------------------------------------------ */
/* The trajectory scoring of DetZero's training-target assignment (target_assign.assign_track_target,
 * tracking/detzero_track/models/tracking_modules/target_assign.py:8-139; recall = 0, BEV IoU) and of its tracklet recall
 * (TrackRecall.eval_single_seq, tracking/detzero_track/utils/track_recall.py:153-262 with get_trajectory_similarity of
 * utils/track_calculation.py:84-123; recall = 1, 3-D IoU when iou_3d), for S sequences in one launch.
 * Ground truth: gt_box (S, F, G, 7) float32 lidar boxes, gt_world (S, F, G, 9) float64 world boxes, gt_cls (S, F, G) class 1..3 or 0
 * (never scored), gt_obj the per-sequence object index (0 .. n_obj[s] - 1, -1 for a class-0 row), gt_diff / gt_npts difficulty and
 * num_points_in_gt, gt_cnt (S, F) rows per frame, gt_num_frames (S).  Tracks: the dz_track_sequences outputs trk (S, max_tracks, 6),
 * n_tracks, ent_box (S, max_entries, 9), ent_frame, and poses (S, F, 4, 4) lidar -> world of the same frames.
 * thresholds (3 doubles): the IoU threshold per class; class_mask: bit c set when class c is scored.
 * Outputs: obj_rec (S, max_objects, 5) int32 [matched track or -1, match count, trajectory length, bucket 1 (L1) / 2 (L2), class];
 * trk_rec (S, max_tracks, 4) int32 [matched object or -1, class, entry count, dynamic]; ent_iou (S, max_entries) float32 the BEV IoU
 * of each entry with its track's matched object in that frame (0 where absent); overflow[s] != 0 when the max_pairs pair table or the
 * assignment scratch overflowed (the sequence's outputs are then invalid).  One block per sequence, no host synchronisation. */
size_t dz_track_gt_ws_bytes(int S, int F, int max_objects, int max_tracks, int max_entries, int max_pairs);
int dz_track_gt(const float* gt_box, const double* gt_world, const int* gt_cls, const int* gt_obj, const int* gt_diff, const int* gt_npts,
                const int* gt_cnt, const int* gt_num_frames, const int* n_obj, int S, int F, int G, int max_objects, const int* trk,
                const int* n_tracks, const double* ent_box, const int* ent_frame, const double* poses, int max_tracks,
                int max_entries, const double* thresholds, int class_mask, int recall, int iou_3d, int max_pairs, int* obj_rec,
                int* trk_rec, float* ent_iou, int* overflow, void* ws, size_t ws_bytes, dz_stream_t stream);

/* ---- refiner inputs (SURVEY.md 8f row 2), csrc/refine_data.cu -------------------------------------------------------------- */
/* Builds the eval inputs of the refiner modules for B tracks of up to L box slots straight from the collated frames, in one call per
 * kind: PRM (kind 0) = WaymoPositionDataset.extract_track_feature (refining/detzero_refine/datasets/waymo/waymo_position_dataset.py:31-184),
 * CRM (kind 1) = WaymoConfidenceDataset.extract_track_feature (waymo_confidence_dataset.py:59-162), GRM (kind 2) =
 * WaymoGeometryDataset.extract_track_feature (waymo_geometry_dataset.py:26-154), fused with the object crop of
 * daemon/prepare_object_data.py:241-327 (enlarged boxes, roiaware_pool3d_kernel.cu:23-36 test) and sample_points
 * (refining/detzero_refine/utils/data_utils.py:12-30).  The sampling is keyed and deterministic and the geometry float64: see the
 * header of csrc/refine_data.cu for the exact key function and the other deliberate deviations.
 *   points (rows of pt_stride >= 5 floats [b, x, y, z, tanh(i), ...], lidar frame) with frame_offsets (n_frames + 1); max_frame_points
 *   (host) >= the largest frame.  poses (n_frames, 4, 4) f64 lidar -> world.  Tracks: boxes (B, L, 7) f64 world, frame_of_box (B, L),
 *   scores (B, L) f32, box_num (B) (1..L), cls (B) (1-based, the cyclist one-hot), track_uid (B) i64.
 *   crop = 0: every point of the box's frame belongs to the box (per-object point sets packed one frame per box).
 *   kq / km / nq: query points, memory points, GRM query boxes (QUERY_POINTS_NUM, MEMORY_POINTS_NUM, QUERY_NUM).
 * Outputs (f32 unless noted), PRM: q_pts (B, L, kq, C) pos_query_points, m_pts (B, L, km, C) pos_memory_points, C = 32 (+3 with_class),
 *   traj (B, L, 7) pos_trajectory, box_f (B, L) padding_mask, track_f (B, 7) pos_init_box.  CRM: q_pts (B, L, kq, 32) conf_points,
 *   box_f (B, L) conf_score (-1 padded).  GRM: q_pts (B, q_out, kq, 4) geo_query_points, m_pts (B, km, 11) geo_memory_points,
 *   traj (B, L, 7) world boxes, box_f (B, q_out, 7) geo_query_boxes, query_num (B) int32 geo_query_num.
 *   counts (B, L) int32 crop counts and sel (the sorted selected ranks: PRM (B, L, kq + km), CRM (B, L, kq), GRM (B, nq * kq + km))
 *   are optional outputs (NULL: kept in the workspace). */
size_t dz_refine_inputs_ws_bytes(int kind, int B, int L, int max_frame_points, int kq, int km, int nq);
int dz_refine_inputs(int kind, const float* points, int pt_stride, const int32_t* frame_offsets, int n_frames, int max_frame_points,
                     const double* poses, const double* boxes, const int32_t* frame_of_box, const float* scores,
                     const int32_t* box_num, const int32_t* cls, const int64_t* track_uid, int B, int L, int kq, int km, int nq,
                     int q_out, int with_class, double enlarge_scale, int crop_on_bev, int crop, unsigned long long seed,
                     float* q_pts, float* m_pts, float* traj, float* box_f, float* track_f, int32_t* query_num, int32_t* counts,
                     int32_t* sel, void* ws, size_t ws_bytes, dz_stream_t stream);
/* revert_to_each_frame: PRM (kind 0) pred (B, L, 7) in the init-box frame -> world (box_coords_transform, data_utils.py) -> lidar
 * (world_to_lidar) (waymo_position_dataset.py:257-286); GRM (kind 2) pred (B, 7): its size written into each world box -> lidar
 * (waymo_geometry_dataset.py:160-186).  lidar, world (B, L, 7) f64, rows past box_num zero. */
int dz_refine_revert(int kind, const float* pred, const double* poses, int n_frames, const double* boxes, const int32_t* frame_of_box,
                     const int32_t* box_num, int B, int L, double* lidar, double* world, dz_stream_t stream);

/* ---- combine: refined tracks -> per-frame result rows (csrc/combine.cu) ------------------------------------------------------- */
/* convert_frame_format + combine_det as combine_final drives them (daemon/combine_output.py:27-41,44-99,102-167), for the B tracks
 * of one sequence in output order: prm_lidar (B, L, 7) f64 (revert_position_boxes' lidar boxes), grm_pred (B, 7) f32 (only its size
 * is read; the reference reads the same bits from the GRM's reverted boxes), score (B, L) f32 (CRM pred_score, or the tracker's
 * per-box score), frame_of_box (B, L) (0..F-1), box_num (B) (0..L), cls (B) (label), track_id (B) (>= 0).  Optional (det NULL: none)
 * the tracker's dropped detections: det (F, K, 9) f32 gathered rows, det_count (F), kept (F, K) u8 (TrackResult.kept).
 * Outputs: rows (F, R, 9) f32 [x, y, z, dx, dy, dz, heading, score, label], obj_id (F, R) (-1 for a dropped detection), count (F);
 * rows of a frame: its track boxes by track then box order, then its dropped rows in input order with det_drop's heading wrap.
 * A frame without a track box gets no row (combine_det only extends frames convert_frame_format emitted).  Rows past count[f] are
 * not written.  overflow (zeroed by the caller): bit 1 = a frame needed more than R rows (count clamped, nothing written past R),
 * bit 2 = a frame index outside 0..F-1 (box skipped).  Deterministic (no atomic places a row), enqueue only.
 * Deviations from combine_final: the reference writes one file per class and its class loop accumulates (each file holds every
 * class processed so far; the last one omits sequences without a track of the last class); here one call combines the given tracks,
 * every class at once.  combine_det raises KeyError for a frame with tracks but no drop entry; here that frame has no dropped row. */
size_t dz_combine_frames_ws_bytes(int B, int L, int F);
int dz_combine_frames(const double* prm_lidar, const float* grm_pred, const float* score, const int32_t* frame_of_box,
                      const int32_t* box_num, const int32_t* cls, const int32_t* track_id, int B, int L, const float* det,
                      const int32_t* det_count, const unsigned char* kept, int K, int F, int R, float* rows, int32_t* obj_id,
                      int32_t* count, int32_t* overflow, void* ws, size_t ws_bytes, dz_stream_t stream);

/* ---- the refiners against ground truth (csrc/refine_gt.cu) --------------------------------------------------------------------- */
/* Ground truth per track slot, for B tracks of one sequence with L box slots (daemon/prepare_object_data.py:64-190, which attaches
 * gt_boxes_global / matched / matched_tracklet / state to each track box on the host, and the gt_pos_trajectory of
 * refining/detzero_refine/datasets/waymo/waymo_position_dataset.py:41-42,76-80,159-160).  gt_world (F, G, 9) f64, gt_obj (F, G),
 * gt_cnt (F): one sequence of the dz_track_gt ground-truth tables.  trk_obj (B): the object matched to each track (dz_track_gt's
 * trk_rec[.., 0]) or -1; obj_state / trk_state (B): the matched object's state (trk_rec[.., 3]) and the tracker's own (trk[.., 4]).
 * boxes (B, L, 7) f64 world, frame_of_box (B, L), box_num (B): the track tables of dz_refine_inputs.
 * Outputs: gt_boxes (B, L, 7) f64 world, the matched object's box in the slot's frame (its first row there), zeros where it has none,
 * for an unmatched track and past box_num; matched (B, L) u8: 1 where the object is present, and 1 on every valid slot of an
 * unmatched track (prepare_object_data.py:184-188); matched_tracklet (B) u8; state (B) (1 dynamic): the object's for a matched
 * track, the tracker's otherwise; gt_traj (B, L, 7) f32: gt_boxes in the frame of the track's init box (slot box_num / 2), by the
 * float64 transform dz_refine_inputs kind 0 applies to pos_trajectory (zero boxes included, as init_coords_transform does), rows
 * past box_num zero. */
int dz_refine_targets(const double* gt_world, const int32_t* gt_obj, const int32_t* gt_cnt, int F, int G, const int32_t* trk_obj,
                      const int32_t* obj_state, const int32_t* trk_state, const double* boxes, const int32_t* frame_of_box,
                      const int32_t* box_num, int B, int L, double* gt_boxes, unsigned char* matched,
                      unsigned char* matched_tracklet, int32_t* state, float* gt_traj, dz_stream_t stream);
/* out[i] = 3-D IoU of boxes_a[i] and boxes_b[i] (rows of >= 7 floats, row strides lda / ldb): the diagonal of dz_boxes_pairwise
 * kind 2, bit for bit.  Replaces iou3d_nms_utils.boxes_iou3d_gpu(a, b).diag(), which computes n x n rotated clips to keep n. */
int dz_boxes_iou3d_aligned(const float* boxes_a, int lda, const float* boxes_b, int ldb, int n, float* out, dz_stream_t stream);
/* The per-box IoUs and per-track counts of generate_recall_record (refining/detzero_refine/models/position_refine_model.py:100-133,
 * geometry_refine_model.py:98-141), one block per track, one launch: in_boxes / out_boxes / gt_boxes (B, L, 7) f64 world (the box
 * before and after refinement, and dz_refine_targets' gt_boxes), size (B, 7) f32 or NULL: when given, the refined box takes its
 * dx, dy, dz from size[b][3:6] (the GRM's prediction, geometry_refine_model.py:105-108).  Every pair is re-centred on its ground-truth
 * centre in float64, rounded to float32 and clipped as dz_boxes_pairwise kind 2 does.  A slot is scored when matched_tracklet[b] and
 * matched[b][j] and j < box_num[b].  thresholds: n_thresholds <= 8 host doubles, compared as float32 (iou > th).
 * Outputs: iou_in, iou_out (B, L) f32 (0 on the slots not scored); rec (B, 1 + 2 n) int32 [scored slots, count(iou_in > th_k)..,
 * count(iou_out > th_k)..].  A ground-truth box without volume gives 0.
 * out_boxes == NULL is label mode, generate_refine_boxes_iou (daemon/generate_iou_gt.py:36-53): every slot below box_num is scored,
 * in_boxes (with size, when given) against gt_boxes; only iou_in (and rec, when not NULL) is written. */
int dz_refine_score(const double* in_boxes, const double* out_boxes, const float* size, const double* gt_boxes,
                    const unsigned char* matched, const unsigned char* matched_tracklet, const int32_t* box_num, int B, int L,
                    const double* thresholds, int n_thresholds, float* iou_in, float* iou_out, int32_t* rec, dz_stream_t stream);
/* The CRM counters (confidence_refine_model.py:81-104) per track over its box_num slots, from conf_score, pred_score, iou (B, L) f32:
 * rec (B, 5) int32 [matched_up, matched_down, unmatched_up, unmatched_down, box_num] with gt_label = iou >= 0.7 (float32) and
 * up = pred_score >= conf_score. */
int dz_confidence_score(const float* conf_score, const float* pred_score, const float* iou, const int32_t* box_num, int B, int L,
                        int32_t* rec, dz_stream_t stream);

/* ---- detection AP / APH records (csrc/det_eval.cu) --------------------------------------------------------------------------- */
/* The per-cutoff counts behind Waymo AP and APH as DetZero's evaluator reports them (evaluator/detzero_eval.py ->
 * WaymoDetectionMetricsEstimator), restated without the Waymo metric library (the definition is in csrc/det_eval.cu).
 * pred (NF, R, 9) f32 [x, y, z, dx, dy, dz, heading, score, Waymo type] with pred_cnt (NF) rows per frame; gt_box (NF, G, 7) f32,
 * gt_type (NF, G) Waymo type, gt_level (NF, G) 1 or 2, gt_cnt (NF).  Waymo types are 1 vehicle, 2 pedestrian, 3 sign, 4 cyclist;
 * a row of any other type is ignored.  box_type 0: 3-D IoU (boxes_iou3d_gpu), 1: BEV IoU.  breakdown_mask bit 0: OBJECT_TYPE
 * (records shards 0..3, type - 1), bit 1: RANGE (shards 4..15, 4 + 3 (type - 1) + range, range [0, 30) / [30, 50) / [50, +inf)).
 * records (16, 2, 101, 4) int64 [shard][LEVEL_1, LEVEL_2][cutoff k: score >= float32(k * 0.01), the last 1.0][TP, FP, FN, TPH
 * (2^-32 units)] are ADDED to (the caller zeroes them once; records of disjoint frame sets add up); shards outside the mask are not
 * written.  *overflow (zeroed by the caller) gets bit 1 when a frame has more than max_pairs valid pairs, bit 2 when an assignment
 * component exceeds the scratch; the records are then invalid.  Persistent blocks, integer atomics (the records are identical run to
 * run), no host synchronisation. */
size_t dz_det_eval_ws_bytes(int NF, int R, int G, int max_pairs);
int dz_det_eval(const float* pred, const int* pred_cnt, const float* gt_box, const int* gt_type, const int* gt_level, const int* gt_cnt,
                int NF, int R, int G, int box_type, int breakdown_mask, int max_pairs, long long* records, int* overflow, void* ws,
                size_t ws_bytes, dz_stream_t stream);

/* ---- tracking MOTA / MOTP records (csrc/track_eval.cu) ---------------------------------------------------------------------- */
/* The per-cutoff counts behind Waymo MOTA, MOTP, MISS, MISMATCH and FP as DetZero's evaluator reports them in tracking mode
 * (evaluator/detzero_eval.py --tracking -> WaymoTrackingMetricsEstimator), restated as CLEAR-MOT without the Waymo metric library
 * (the definition is in csrc/track_eval.cu).  Per-sequence padded tables: pred (S, F, R, 9) f32 [x, y, z, dx, dy, dz, heading,
 * score, Waymo type], pred_id (S, F, R) int32 identity per sequence, pred_cnt (S, F); gt_box (S, F, G, 7) f32, gt_obj (S, F, G)
 * object index in [0, n_obj[s]), gt_type (S, F, G) Waymo type (any other type: the row is ignored), gt_level 1 or 2, gt_cnt (S, F);
 * num_frames (S) frames per sequence, in order; max_objects >= every n_obj.  breakdown_mask bit 0 OBJECT_TYPE, bit 1 RANGE (shards
 * as dz_det_eval).  records (16, 2, 101, 5) int64 [shard][LEVEL_1, LEVEL_2][cutoff][matches, misses, FP, mismatches, cost (2^-32
 * units)] are ADDED to (records of disjoint sequence sets add up).  *flags (zeroed by the caller): bit 1 a frame has more than
 * max_pairs valid pairs of one type, bit 2 an assignment component exceeds the scratch (the records are then invalid), bit 4 two
 * rows of a frame share an id, bit 8 an object index is out of range.  One block per (type, sequence), integer atomics (identical
 * run to run), no host synchronisation. */
size_t dz_track_eval_ws_bytes(int S, int R, int G, int max_objects, int max_pairs);
int dz_track_eval(const float* pred, const int* pred_id, const int* pred_cnt, const float* gt_box, const int* gt_obj, const int* gt_type,
                  const int* gt_level, const int* gt_cnt, const int* num_frames, const int* n_obj, int S, int F, int R, int G,
                  int max_objects, int breakdown_mask, int max_pairs, long long* records, int* flags, void* ws, size_t ws_bytes,
                  dz_stream_t stream);
/* Track entries back to the lidar frame as dz_track_gt does (transform_boxes3d(inverse=True) of convert_frame_format): ent_box
 * (S, E, 9) f64 world boxes, ent_frame (S, E), poses (S, F, 4, 4) lidar -> world, num_frames (S) -> out (S, E, 7) f32 (zeros for an
 * entry whose frame is not in [0, num_frames[s])). */
int dz_track_entry_lidar(const double* ent_box, const int* ent_frame, const double* poses, const int* num_frames, int S, int E, int F,
                         float* out, dz_stream_t stream);

/* ---- test-time augmentation (CenterPoint TTA) ------------------------------------------------------------- */
/* A view is 4 host floats [op, p1, p2, p3]: DZ_TTA_ORIGINAL; DZ_TTA_FLIP_X (y = -y); DZ_TTA_FLIP_Y (x = -x); DZ_TTA_FLIP_XY;
 * DZ_TTA_ROT with p1, p2 = cos, sin of the float32 angle (float32 torch on the CPU, as the reference computes them) and, for
 * dz_tta_unaugment only, p3 = the float32 heading offset; DZ_TTA_SCALE with p1 = the float32 scale. */
enum { DZ_TTA_ORIGINAL = 0, DZ_TTA_FLIP_X = 1, DZ_TTA_FLIP_Y = 2, DZ_TTA_FLIP_XY = 3, DZ_TTA_ROT = 4, DZ_TTA_SCALE = 5 };
enum { DZ_TTA_MAX_VIEWS = 32, DZ_WBF_MAX_LABELS = 8 };
/* points (N, stride) collated [b, x, y, z, feats...], frames contiguous with host-known sizes h_frame_sizes (B) ->
 * out (V*N, stride): frame b view v at rows V*start_b + v*n_b .. with batch index b*V + v, x/y/z augmented, features copied.
 * Replaces TestTimeAugmentor.forward (detection/detzero_det/datasets/augmentor/test_time_augmentor.py:32-100, rotation by
 * common_utils.rotate_points_along_z, utils/detzero_utils/common_utils.py:220-244) and the TTA branch of collate_batch
 * (detection/detzero_det/datasets/dataset.py:260-303), which build the views in numpy in the DataLoader workers. */
int dz_tta_expand(const float* points, int stride, const int* h_frame_sizes, int B, const float* h_views, int V, float* out,
                  dz_stream_t stream);
/* boxes (BV, K, 9) [x,y,z,dx,dy,dz,heading,score,label] with counts (BV,) -> out (BV, K, 9) in the original frame (inverse of view
 * bv % V; rows past the count are zeroed).  Replaces the restore loop of CenterPoint.test_time_augment
 * (detection/detzero_det/models/centerpoint.py:157-202). */
int dz_tta_unaugment(const float* boxes, const int* counts, int BV, int K, const float* h_views, int V, float* out,
                     dz_stream_t stream);
/* 3-D weighted box fusion of the V views of each of B frames: boxes (B*V, K, 9) + counts (B*V,) -> out (B, V*K, 9) fused rows
 * [x,y,z,dx,dy,dz,heading,score,label] in descending score order (ties: the cluster's first member by (view, row)), out_count (B,).
 * Labels 1..L with h_iou_thr / h_skip_thr (host, L doubles, indexed label-1); other labels are dropped.  conf_type 'avg', unit
 * weights, allows_overflow False.  V*K <= 16384.  Replaces weighted_boxes_fusion_3d
 * (detection/detzero_det/utils/ensemble_utils/wbf_3d.py:10-190) as called by wbf_online (ensemble.py:7-32), whose
 * find_matching_box launches boxes_iou3d_gpu and reads the IoU back once per input box. */
size_t dz_wbf_3d_ws_bytes(int B, int V, int K, int L);
int dz_wbf_3d(const float* boxes, const int* counts, int B, int V, int K, const double* h_iou_thr, const double* h_skip_thr, int L,
              float* out, int* out_count, void* ws, size_t ws_bytes, dz_stream_t stream);

/* ---- refiner (GRM / PRM / CRM)------------------------------------------------------------------------- */
/* y = act((x @ W^T) * scale + shift): x (M,K) row-major, W (N,K) row-major (nn.Linear / 1x1 Conv layout).
 * Replaces F.linear and the Conv1d/Conv2d(k=1)+BN+ReLU MLP stacks (utils/detzero_utils/model_utils.py:81-134). */
int dz_linear_fwd(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift,
                  int relu, float* y, int ldy, int mode, dz_stream_t stream);
/* The same with a per-row-GROUP shift: y[m] = act((x[m] W^T) * scale + shift + gshift[m / gsize]), gshift (M/gsize, N).  Serves the
 * PointNet "concatenate the max-pooled global feature back onto every point, then Linear" step (position_transformer.py:118-123,
 * geometry_transformer.py:131-136, confidence_pointnet.py:88-100) without materialising the concatenation: W = [W_g | W_p],
 * gshift = (g W_g^T) * scale computed once per group, x = the per-point half. */
int dz_linear_fwd_grouped(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift,
                          const float* gshift, int gsize, int relu, float* y, int ldy, int mode, dz_stream_t stream);
/* Linear (+folded BN +ReLU) fused with the max over groups of `group` consecutive rows (group % 128 == 0, K % 32 == 0, N % 4 == 0,
 * tensor-core mode): y (M/group, N).  The last layer of a PointNet encoder + torch.max over the points in one kernel. */
int dz_linear_max_fwd(const float* x, int M, int K, const float* w, int N, const float* scale, const float* shift, int relu,
                      int group, float* y, int mode, dz_stream_t stream);
/* max over `group` consecutive rows: x (G*group, C) -> y (G, C)  (torch.max over points,
 * position_transformer.py:109,118) */
int dz_group_max(const float* x, int G, int group, int C, float* y, dz_stream_t stream);
/* softmax(q k^T + key_padding) v per (batch, head); q already scaled.  q (B,Pq,H*dh), k/v (B,Pk,H*dh) with
 * row strides ldq/ldk/ldv ; key_padding_mask (B,Pk) u8 (non-zero = masked, as masked_fill(-inf)) or NULL.
 * Replaces multi_head_attention.py:266-286 without materialising the (B*H,Pq,Pk) score tensor. */
int dz_attention_fwd(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                     const unsigned char* key_padding_mask, int B, int Pq, int Pk, int H, int dh, float* out,
                     int ldo, int mode, dz_stream_t stream);
/* ConfidencePointnet point encoders in TRAIN mode, forward and backward, recomputing the point layers tile by tile instead of storing
 * them (confidence_pointnet.py:80-92 with BatchNorm2d batch statistics, and the autograd backward of those lines).  One pass over the
 * x (crops*P, c0) point rows, P % 64 == 0, c0 % 8 == 0 and <= 64, layers c0 -> 128 -> 128 -> 256 and [g | y2] 384 -> 256:
 *   1..4  sums of z_l and z_l^2 of layer l -> stats[0..256), stats[256..512) (float64); 3 and 4 also: zext / iext (2, crops, 256) the
 *         max / min z over each crop and their lowest row in the crop; 4 also csum (crops, 256), the crop sums of z4
 *   5     slab (2, 256, 128) = dW4p, dW3 (float64); stats = sum dh2, sum dh2 * xhat2
 *   6     slab (128, 128) = dW2; stats = sum dh1, sum dh1 * xhat1
 *   7     slab (128, c0) = dW1
 * w*t: forward weights transposed (K x N); w2, w3, w4p: as stored (N x K), w4p = the last 128 input columns of pts_encoder_2's weight.
 * tab (4, 6, 256): per layer and channel [a = gamma*rstd, b = beta - mean*a, mean, rstd, m1 = sum dh / N, m2 = sum dh*xhat / N];
 * shift4 (crops, 256) = g W4g^T; sel / dsel (2, crops, 256): the pooled row and dL/dh there, layer 3 then layer 4.  Partials are
 * per CTA and reduced in a fixed order: the same inputs give the same bits.  mode DZ_F32 (fp32 FMA) or DZ_TF32 (TF32 tensor cores). */
size_t dz_crm_point_ws_bytes(int crops);
int dz_crm_point_pass(int pass, int mode, const float* x, int crops, int P, int c0, const float* w1t, const float* w2t,
                      const float* w3t, const float* w4pt, const float* w2, const float* w3, const float* w4p, const float* tab,
                      const float* shift4, const int* sel, const float* dsel, float* zext, int* iext, double* csum, double* stats,
                      double* slab, void* ws, size_t ws_bytes, dz_stream_t stream);
/* y = LayerNorm(x + r) * gamma + beta over the last dim C (decoder.py:73-75,85-90) ; r may be NULL */
int dz_layernorm_residual(const float* x, const float* r, const float* gamma, const float* beta, float eps,
                          int M, int C, float* y, dz_stream_t stream);

/* out = a + b, n % 4 == 0 (with_pos_embed, decoder.py:45-46) */
int dz_add(const float* a, const float* b, size_t n, float* out, dz_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif

"""Float64 numpy restatement of the refiner input builder (detzero_b200/csrc/refine_data.cu, detzero_b200/refine/data.py): the
per-object crop, the keyed sampler, the PRM / CRM / GRM encodings of the eval branch and the revert of refined boxes to each frame.

Reference: daemon/prepare_object_data.py:241-327 (crop), refining/detzero_refine/utils/data_utils.py (sample_points,
init_coords_transform, local_coords_transform, box_coords_transform, world_to_lidar), WaymoPositionDataset /
WaymoGeometryDataset / WaymoConfidenceDataset.extract_track_feature and revert_to_each_frame.

Deliberate deviations from the reference (the same list is in the header comment of csrc/refine_data.cu):
  1. Sampling is deterministic.  ``sample_points`` calls random.sample; here a selection of k of n candidates keeps the k ranks with
     the smallest keys  key(r) = mix64(base + r),  base = mix64(mix64(mix64(seed) ^ track_uid) ^ (box_slot << 8 | stream)),  all
     arithmetic mod 2^64, mix64 = the splitmix64 step (add 0x9E3779B97F4A7C15, then the two xor-shift-multiply rounds and the final
     xor-shift).  mix64 is a bijection, so the keys of one selection are distinct; the selected ranks are returned sorted.  That is a
     uniform k-subset in sorted order, as the reference draws, and a track's inputs depend on (seed, track_uid) only.  Streams:
     PRM query 0, PRM memory 1, CRM 2, GRM query 3 (slot = the query box), GRM memory 4 (slot 0, over the track's concatenation).
  2. Geometry is float64 throughout (the reference rounds its trajectory and rotation matrices to float32).
  3. GRM's query count is min(QUERY_NUM, L) per track (the reference lowers self.query_num for every later track).
  4. The crop tests each point of the box's lidar frame in float64 world coordinates taken relative to the box centre
     (pose applied to the float32 lidar point), where the reference tests float32 world points.  Only points within about 1e-3 m
     of an enlarged face can land differently.
"""
import numpy as np

PRM_Q, PRM_M, CRM_Q, GRM_Q, GRM_M = 0, 1, 2, 3, 4
M64 = (1 << 64) - 1
GAMMA = 0x9E3779B97F4A7C15
CORNERS = np.array([[1, 1, -1], [1, -1, -1], [-1, -1, -1], [-1, 1, -1],
                    [1, 1, 1], [1, -1, 1], [-1, -1, 1], [-1, 1, 1]], np.float64) / 2      # box_utils.boxes_to_corners_3d


def mix64_int(z):
    z = (int(z) + GAMMA) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def mix64(z):
    """vectorised mix64 on uint64 arrays (wrapping arithmetic)"""
    z = np.asarray(z, np.uint64)
    with np.errstate(over='ignore'):
        z = z + np.uint64(GAMMA)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def key_base(seed, uid, slot, stream):
    return mix64_int(mix64_int(mix64_int(seed) ^ (int(uid) & M64)) ^ ((int(slot) << 8) | int(stream)))


def sample_ranks(n, k, seed, uid, slot, stream):
    """sorted ranks of the k smallest keys among ranks 0..n-1 (all n ranks when n <= k)"""
    if n <= k:
        return np.arange(n, dtype=np.int64)
    with np.errstate(over='ignore'):
        keys = mix64(np.uint64(key_base(seed, uid, slot, stream)) + np.arange(n, dtype=np.uint64))
    return np.sort(np.argpartition(keys, k - 1)[:k]).astype(np.int64)


def limit_heading(a):
    """data_utils.limit_heading_range on one value: into [-pi, pi)"""
    a = float(a)
    while a >= np.pi:
        a -= 2 * np.pi
    while a < -np.pi:
        a += 2 * np.pi
    return a


def rz(a):
    """rotation by +a about z (x -> y)"""
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def crop_box(frame_pts, pose, box, enlarge=1.1, bev=False, crop=True):
    """(n, >=4) f32 lidar rows [x, y, z, tanh(i), ...] of the box's frame -> (m, 4) float64 [world xyz - box centre, tanh(i)] of the
    points inside the enlarged box, in frame order (prepare_object_data.py:249-311 with the in/out test of
    roiaware_pool3d_kernel.cu:23-36: x/y margin 1e-5, none on z)"""
    p = np.asarray(frame_pts[:, :3], np.float64)
    rel = p @ pose[:3, :3].T + (pose[:3, 3] - box[:3])
    if crop:
        dx, dy, dz = box[3] * enlarge, box[4] * enlarge, (100.0 if bev else box[5] * enlarge)
        c, s = np.cos(-box[6]), np.sin(-box[6])
        lx, ly = rel[:, 0] * c - rel[:, 1] * s, rel[:, 0] * s + rel[:, 1] * c
        m = (np.abs(rel[:, 2]) <= dz / 2) & (np.abs(lx) < dx / 2 + 1e-5) & (np.abs(ly) < dy / 2 + 1e-5)
    else:
        m = np.ones(len(p), bool)
    return np.concatenate([rel[m], np.asarray(frame_pts[m, 3:4], np.float64)], 1)


def track_crops(frames, frame_offsets, poses, boxes, fob, L, enlarge=1.1, bev=False, crop=True):
    """per box of one track: the cropped rows of crop_box"""
    out = []
    for j in range(L):
        f = int(fob[j])
        out.append(crop_box(frames[frame_offsets[f]:frame_offsets[f + 1], 1:5], poses[f], boxes[j], enlarge, bev, crop))
    return out


def _pad(rows, k):
    o = np.zeros((k, rows.shape[1]))
    o[:len(rows)] = rows
    return o


def init_frame(boxes, L):
    """init_coords_transform: init box (heading wrapped), and the trajectory in the init-box frame"""
    init = boxes[L // 2].copy()
    init[6] = limit_heading(init[6])
    R = rz(-init[6])
    traj = boxes[:L].copy()
    traj[:, :3] = (traj[:, :3] - init[:3]) @ R.T
    traj[:, 6] = [limit_heading(limit_heading(h) - init[6]) for h in boxes[:L, 6]]
    return init, R, traj


def corners_centre(box):
    """(9, 3): the 8 corners of boxes_to_corners_3d, then the centre"""
    c = (box[3:6] * CORNERS) @ rz(box[6]).T + box[:3]
    return np.concatenate([c, box[None, :3]], 0)


def encode_p2co(pts, box, score, cls_onehot):
    """[xyz, intensity, p2co (27), score (, class)] of (k, 4) rows in the init-box frame (zero rows included)"""
    cc = corners_centre(box).reshape(-1)
    cols = [pts[:, :3], pts[:, 3:4], np.tile(pts[:, :3], (1, 9)) - cc[None, :], np.full((len(pts), 1), score)]
    if cls_onehot is not None:
        cols.append(np.tile(cls_onehot[None, :], (len(pts), 1)))
    return np.concatenate(cols, 1)


def _onehot(cls, with_class):
    if not with_class:
        return None
    o = np.zeros(3)
    o[int(cls) - 1] = 1
    return o


def position_track(crops, boxes, scores, L, cls, uid, seed, Lmax=200, kq=256, km=48, with_class=False):
    """WaymoPositionDataset.extract_track_feature (eval) for one track; crops = track_crops(...)"""
    init, R, traj = init_frame(boxes, L)
    oh = _onehot(cls, with_class)
    C = 32 + (3 if with_class else 0)
    q = np.zeros((Lmax, kq, C))
    m = np.zeros((Lmax, km, C))
    sel_q, sel_m = [], []
    for j in range(L):
        local = crops[j].copy()
        local[:, :3] = (local[:, :3] + (boxes[j, :3] - init[:3])) @ R.T
        sq = sample_ranks(len(local), kq, seed, uid, j, PRM_Q)
        sm = sample_ranks(len(local), km, seed, uid, j, PRM_M)
        sel_q.append(sq)
        sel_m.append(sm)
        q[j] = encode_p2co(_pad(local[sq], kq), traj[j], scores[j], oh)
        m[j] = encode_p2co(_pad(local[sm], km), traj[j], scores[j], oh)
    tr = np.zeros((Lmax, 7))
    tr[:L] = traj
    mask = np.ones(Lmax)
    mask[:L] = 0
    return {'pos_query_points': q, 'pos_memory_points': m, 'pos_trajectory': tr, 'padding_mask': mask, 'pos_init_box': init,
            'box_num': L, 'sel': (sel_q, sel_m)}


def confidence_track(crops, boxes, scores, L, uid, seed, Lmax=200, kq=256):
    """WaymoConfidenceDataset.extract_track_feature (eval) for one track"""
    init, R, traj = init_frame(boxes, L)
    q = np.zeros((Lmax, kq, 32))
    sel = []
    for j in range(L):
        local = crops[j].copy()
        local[:, :3] = (local[:, :3] + (boxes[j, :3] - init[:3])) @ R.T
        s = sample_ranks(len(local), kq, seed, uid, j, CRM_Q)
        sel.append(s)
        q[j] = encode_p2co(_pad(local[s], kq), traj[j], scores[j], None)
    cs = np.full(Lmax, -1.0)
    cs[:L] = scores[:L]
    return {'conf_points': q, 'conf_score': cs, 'box_num': L, 'sel': sel}


def query_order(scores, L, nq=3):
    """np.argsort(score)[::-1][:nq] with ties broken by the later index first"""
    return [int(j) for j in sorted(range(L), key=lambda j: (-float(scores[j]), -j))[:min(nq, L)]]


def geometry_track(crops, boxes, scores, L, uid, seed, nq=3, kq=256, km=4096):
    """WaymoGeometryDataset.extract_track_feature (eval) for one track: query points / boxes of the top-scored boxes, memory
    sampled from the concatenation of every box's encoded points"""
    qidx = query_order(scores, L, nq)
    local, enc = [], []
    for j in range(L):
        p = crops[j].copy()
        p[:, :3] = p[:, :3] @ rz(-boxes[j, 6]).T
        local.append(p)
        h = boxes[j, 3:6] / 2
        enc.append(np.concatenate([p[:, :3], p[:, 3:4], h - p[:, :3], h + p[:, :3], np.full((len(p), 1), scores[j])], 1))
    allp = np.concatenate(enc, 0) if enc else np.zeros((0, 11))
    sm = sample_ranks(len(allp), km, seed, uid, 0, GRM_M)
    mem = _pad(allp[sm], km)
    qp = np.zeros((len(qidx), kq, 4))
    qb = np.zeros((len(qidx), 7))
    sel_q = []
    for i, j in enumerate(qidx):
        s = sample_ranks(len(local[j]), kq, seed, uid, j, GRM_Q)
        sel_q.append(s)
        qp[i] = _pad(local[j][s], kq)
        qb[i, 3:6] = boxes[j, 3:6]
    return {'geo_query_points': qp, 'geo_query_boxes': qb, 'geo_memory_points': mem, 'geo_query_num': len(qidx),
            'geo_trajectory': boxes[:L].copy(), 'sel': (sel_q, sm), 'query_idx': qidx}


def world_to_lidar(boxes, poses):
    """data_utils.world_to_lidar: per-box inverse pose; heading + atan2(r_t[1,0], r_t[0,0]), not wrapped"""
    out = np.zeros((len(boxes), 7))
    for i, (b, P) in enumerate(zip(boxes, poses)):
        r = np.linalg.inv(P)
        out[i, :3] = r[:3, :3] @ b[:3] + r[:3, 3]
        out[i, 3:6] = b[3:6]
        out[i, 6] = b[6] + np.arctan2(r[1, 0], r[0, 0])
    return out


def revert_position(pred, boxes, L, box_poses):
    """revert_to_each_frame (position): pred (>=L, 7) in the init-box frame -> (lidar (L, 7), world (L, 7))"""
    init, _, _ = init_frame(boxes, L)
    w = np.array(pred[:L], np.float64)
    w[:, :3] = w[:, :3] @ rz(init[6]).T + init[:3]
    w[:, 6] = [limit_heading(h + init[6]) for h in w[:, 6]]
    return world_to_lidar(w, box_poses[:L]), w


def revert_geometry(pred, boxes, L, box_poses):
    """revert_to_each_frame (geometry): the GRM size written into each world box"""
    w = np.array(boxes[:L], np.float64)
    w[:, 3:6] = np.asarray(pred[3:6], np.float64)
    return world_to_lidar(w, box_poses[:L]), w


def build_batch(kind, frames, frame_offsets, poses, tracks, seed, enlarge=1.1, bev=False, crop=True, with_class=False, Lmax=200):
    """every track of a batch; tracks = dict of numpy arrays with the TrackBatch fields.  Returns the list of per-track dicts."""
    out = []
    for b in range(len(tracks['box_num'])):
        L = int(tracks['box_num'][b])
        bx, sc = np.asarray(tracks['boxes'][b], np.float64), np.asarray(tracks['scores'][b])
        crops = track_crops(frames, frame_offsets, poses, bx, tracks['frame_of_box'][b], L, enlarge, bev, crop)
        uid = int(tracks['track_uid'][b])
        if kind == 'prm':
            r = position_track(crops, bx, sc, L, tracks['cls'][b], uid, seed, Lmax, with_class=with_class)
        elif kind == 'crm':
            r = confidence_track(crops, bx, sc, L, uid, seed, Lmax)
        else:
            r = geometry_track(crops, bx, sc, L, uid, seed)
        r['counts'] = np.array([len(c) for c in crops])
        out.append(r)
    return out

"""Device-side pieces of the steps around the detector / refiner (SURVEY.md §8f rows 2, 3), with the reference's function
names so that the tracker / daemon can import them in place of the originals:

  * ``IoUBEV_dis_mat`` / ``IoU3D_dis_mat`` / ``IoU2D_dis_mat`` / ``bev_overlap_gpu`` --
    tracking/detzero_track/models/tracking_modules/data_association/distance.py:44-141.  They take CUDA tensors -- e.g. rows of
    the all-gathered ``(F, 500, 9)`` detection tensor, no ``result.pkl`` hop -- and return CUDA tensors (the reference copies every
    matrix to the host; the Hungarian assignment itself stays on the host and is out of scope).
  * ``points_in_boxes_gpu_v2`` / ``crop_points_in_boxes`` -- utils/detzero_utils/ops/roiaware_pool3d/roiaware_pool3d_utils.py:45-58
    and the per-object crop of daemon/prepare_object_data.py:264-311.
  * ``track_sequences`` -- the whole DetZero tracker (tracking/tools/run_track.py's model forward with its data processor) on the
    device, from the gathered detections of each sequence to post-processed tracks (csrc/tracker.cu).
"""
import ctypes

import numpy as np
import torch

from . import ops
from ._lib import check, darr, lib

IOU_BEV, OVERLAP_BEV, IOU_3D, IOU_2D = 0, 1, 2, 3


def _rows7(t):
    assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.shape[1] >= 7 and t.stride(1) == 1, (t.shape, t.dtype)
    return t


def boxes_pairwise(boxes_a, boxes_b, kind):
    """(N, >=7), (M, >=7) CUDA float rows (any row stride) -> (N, M) CUDA matrix"""
    a, b = _rows7(boxes_a), _rows7(boxes_b)
    out = torch.empty((a.shape[0], b.shape[0]), dtype=torch.float32, device=a.device)
    if a.shape[0] and b.shape[0]:
        check(lib().dz_boxes_pairwise(ops._p(a), a.shape[0], a.stride(0), ops._p(b), b.shape[0], b.stride(0), int(kind), ops._p(out),
                                      ops._stream()), 'boxes_pairwise')
        ops._count(1)
    return out


def IoUBEV_dis_mat(boxes_a, boxes_b, gpu=True):
    return boxes_pairwise(boxes_a, boxes_b, IOU_BEV)


def IoU3D_dis_mat(boxes_a, boxes_b):
    return boxes_pairwise(boxes_a, boxes_b, IOU_3D)


def bev_overlap_gpu(boxes_a, boxes_b):
    return boxes_pairwise(boxes_a, boxes_b, OVERLAP_BEV)


def IoU2D_dis_mat(boxes_a, boxes_b):
    """(N,4), (M,4) [x, y, w, h] like the reference"""
    def pad(t):
        o = torch.zeros((t.shape[0], 7), dtype=torch.float32, device=t.device)
        o[:, 0:2], o[:, 3:5] = t[:, 0:2], t[:, 2:4]
        return o
    return boxes_pairwise(pad(boxes_a), pad(boxes_b), IOU_2D)


dis_mat_dict = {'IoU2D': IoU2D_dis_mat, 'IoU3D': IoU3D_dis_mat, 'IoUBEV': IoUBEV_dis_mat}     # data_association/__init__.py:8-13


def points_in_boxes_gpu_v2(points, boxes):
    """points (B, M, 3), boxes (B, T, 7) -> (B, T, M) int32 mask (the reference's output form)"""
    assert points.shape[0] == boxes.shape[0] and boxes.shape[2] == 7 and points.shape[2] == 3
    out = torch.zeros((points.shape[0], boxes.shape[1], points.shape[1]), dtype=torch.int32, device=points.device)
    for b in range(points.shape[0]):
        p, bx = points[b].contiguous().float(), boxes[b].contiguous().float()
        check(lib().dz_points_in_boxes_mask(ops._p(p), p.shape[0], 3, ops._p(bx), bx.shape[0], 7, ops._p(out[b]), ops._stream()),
              'points_in_boxes_mask')
        ops._count(1)
    return out


def crop_points_in_boxes(points, boxes, cap):
    """points (M, C>=3) [x,y,z,...], boxes (T, >=7) -> idx (T, cap) int32 (indices of each box's points in input order, -1 padded),
    num (T,) int32 true counts.  No (T, M) mask is materialised, nothing goes to the host."""
    assert points.is_cuda and points.dtype == torch.float32 and points.stride(1) == 1
    bx = _rows7(boxes)
    T, M = bx.shape[0], points.shape[0]
    idx = torch.empty((T, cap), dtype=torch.int32, device=points.device)
    num = torch.zeros((T,), dtype=torch.int32, device=points.device)
    if M == 0:
        idx.fill_(-1)
    elif T:
        ws = ops.workspace(lib().dz_crop_points_ws_bytes(M, T), points.device, 'crop')
        check(lib().dz_crop_points_in_boxes(ops._p(points), M, points.stride(0), ops._p(bx), T, bx.stride(0), ops._p(idx), int(cap),
                                            ops._p(num), ops._p(ws), ws.numel(), ops._stream()), 'crop_points_in_boxes')
        ops._count(3)
    return idx, num


CLASS_NAMES = ('Vehicle', 'Pedestrian', 'Cyclist')
#: post-processing steps of the shipped tracker config, in order (box_size_update is commented out there and not supported)
POST_PROCESS = ['empty_track_delete', 'velocity_optimize', 'motion_classify', 'static_drift_eliminate']


def tracker_cfg():
    """tracking/tools/cfgs/tk_model_cfgs/waymo_detzero_track.yaml with tk_dataset_cfgs/waymo_dataset.yaml, per class in CLASS_NAMES
    order: the data processor (heading_process, overlap_box_filter max_score, transform_to_global), the KalmanFilter, two-stage GNN
    association on IoUBEV, track merge, reverse tracking and post-processing"""
    return {'OVERLAP_FILTER': {'METHOD': 'max_score', 'CLASS_THRESHOLD': [0.3, 0.2, 0.2]},
            'FILTER': {'NAME': 'KalmanFilter', 'P': [50, 1000], 'Q': [5, 15], 'R': 0.1, 'DELTA_T': 0.1},
            'TRACK_AGE': {'BIRTH_AGE': 1, 'DEATH_AGE': -1},
            'STAGE': 'two_stage', 'FIRST_STAGE_THRESHOLD': [0.2, 0.1, 0.1], 'SCORE_THRESHOLD': [0.1, 0.1, 0.1],
            'POINT_THRESHOLD': [0, 0, 0], 'SECOND_STAGE_THRESHOLD': [0.3, 0.15, 0.15],
            'MERGE_THRESHOLD': [0.5, 0.4, 0.4], 'REVERSE_TRACKING': True, 'ASSIGN_MODE': False,
            'POST_PROCESS': list(POST_PROCESS), 'LEAST_AGE': 5, 'END_REMOVE': True, 'HEADER_LENGTH': 3}


def _resolve_cfg(cfg):
    c = tracker_cfg()
    if cfg is not None:
        c.update({k: cfg[k] for k in cfg.keys()})
    if c['FILTER']['NAME'] != 'KalmanFilter':
        raise ValueError('filter %r is not supported (KalmanFilter only; AB3DMOT belongs to another config)' % c['FILTER']['NAME'])
    if c['STAGE'] != 'two_stage':
        raise ValueError('association stage %r is not supported (two_stage only)' % c['STAGE'])
    if c['ASSIGN_MODE']:
        raise ValueError('assign_mode (ground-truth target assignment for training) is not supported')
    if list(c['POST_PROCESS']) != POST_PROCESS:
        raise ValueError('post-processing %r is not supported (the shipped list %r only; no box_size_update)' % (c['POST_PROCESS'], POST_PROCESS))
    if c['OVERLAP_FILTER']['METHOD'] != 'max_score' or not c['END_REMOVE'] or not c['REVERSE_TRACKING']:
        raise ValueError('overlap filter max_score, END_REMOVE and REVERSE_TRACKING are required')
    if c['TRACK_AGE'] != {'BIRTH_AGE': 1, 'DEATH_AGE': -1} or any(c['POINT_THRESHOLD']):
        raise ValueError('tracks are born at age 1 and never die, and detections carry no point counts')
    return c


def _params(c):
    f = c['FILTER']
    return darr(list(c['OVERLAP_FILTER']['CLASS_THRESHOLD']) + list(c['FIRST_STAGE_THRESHOLD']) + list(c['SECOND_STAGE_THRESHOLD'])
                + list(c['MERGE_THRESHOLD']) + list(c['SCORE_THRESHOLD']) + list(f['P']) + list(f['Q']) + [f['R'], f['DELTA_T']]
                + [c['LEAST_AGE'], c['HEADER_LENGTH']])


def _yaw_filter(y):
    pi2 = np.float32(np.pi * 2)
    y = np.array(y, np.float32)
    big = np.abs(y) >= pi2
    y[big] = y[big] - np.floor(y[big] / pi2) * pi2
    y[y > np.float32(np.pi)] -= pi2
    y[y <= -np.float32(np.pi)] += pi2
    return y


class TrackResult:
    """Tracks of S sequences (device tensors): trk (S, T, 6) int32 [track id, class 1..3, first frame, entry count, dynamic, entry
    offset] of n_tracks[s] tracks in id order; ent_box (S, E, 9) float64 world boxes [x, y, z, dx, dy, dz, heading, vx, vy],
    ent_score, ent_hit (0 predicted, 1 updated, 2 second-stage match), ent_frame; kept (S, F, K) bool, the overlap filter's keep
    flags of the input rows."""

    def __init__(self, boxes, counts, poses, num_frames, trk, n_tracks, ent_box, ent_score, ent_hit, ent_frame, kept):
        self.boxes, self.counts, self.poses, self.num_frames = boxes, counts, poses, num_frames
        self.trk, self.ent_box, self.ent_score, self.ent_hit, self.ent_frame, self.kept = trk, ent_box, ent_score, ent_hit, ent_frame, kept
        self.n_tracks = n_tracks.cpu().numpy()

    def tracks(self, s=0):
        """(n, 6) int32 host rows of sequence s"""
        return self.trk[s, :int(self.n_tracks[s])].cpu().numpy()

    def track_batch(self, class_name=None, L=200, sequence=0):
        """refine.data.TrackBatch of sequence ``sequence``'s tracks (one class if class_name is given); frame_of_box indexes the
        sequence's frames, track_uid is the track id"""
        from .refine.data import TrackBatch
        t = self.trk[sequence, :int(self.n_tracks[sequence])].long()
        if class_name is not None:
            t = t[t[:, 1] == CLASS_NAMES.index(class_name) + 1]
        cnt = t[:, 3]
        if len(t) and int(cnt.max()) > L:
            raise ValueError('a track has %d boxes (1..%d supported)' % (int(cnt.max()), L))
        ar = torch.arange(L, device=t.device)
        valid = ar[None, :] < cnt[:, None]
        idx = torch.where(valid, t[:, 5:6] + ar[None, :], torch.zeros_like(ar)[None, :])
        boxes = torch.where(valid[..., None], self.ent_box[sequence][idx][..., :7], torch.zeros((), dtype=torch.float64, device=t.device))
        fob = torch.where(valid, self.ent_frame[sequence][idx], torch.zeros((), dtype=torch.int32, device=t.device))
        scores = torch.where(valid, self.ent_score[sequence][idx], torch.zeros((), device=t.device))
        return TrackBatch(boxes, fob, scores, cnt.int(), t[:, 1].int(), t[:, 0], t.device)

    def to_reference(self, sequence_names, frame_ids):
        """(tracks, det_drop) in the form tracking/tools/run_track.py pickles: tracks {seq: {track_id: {'boxes_global', 'name',
        'score', 'sample_idx', 'hit', 'num_points', 'obj_ids', 'pose', 'state'}}}, det_drop {seq: {frame_id: {'boxes_lidar', 'score',
        'name', 'pose', 'frame_id', 'sequence_name'}}}.  frame_ids[s][f] is frame f's id in sequence s."""
        tracks, drops = {}, {}
        boxes, counts, poses, kept = self.boxes.cpu().numpy(), self.counts.cpu().numpy(), self.poses.cpu().numpy(), self.kept.cpu().numpy()
        eb, es, eh, ef = self.ent_box.cpu().numpy(), self.ent_score.cpu().numpy(), self.ent_hit.cpu().numpy(), self.ent_frame.cpu().numpy()
        for s, name in enumerate(sequence_names):
            fids = list(frame_ids[s])
            seq = {}
            for tid, cls, first, cnt, dyn, off in self.tracks(s):
                sl = slice(off, off + cnt)
                seq[int(tid)] = {'boxes_global': eb[s, sl].copy(), 'name': np.array([CLASS_NAMES[cls - 1]] * cnt),
                                 'score': es[s, sl].copy(), 'sample_idx': np.array([fids[f] for f in ef[s, sl]]),
                                 'hit': eh[s, sl].copy(), 'num_points': np.zeros(cnt), 'obj_ids': np.full(cnt, int(tid)),
                                 'pose': poses[s, ef[s, sl]].copy(), 'state': 'dynamic' if dyn else 'static'}
            tracks[name] = seq
            drop = {}
            for f in range(int(self.num_frames[s])):
                n = int(counts[s, f])
                if n == 0:
                    continue
                d = ~kept[s, f, :n]
                lid = boxes[s, f, :n, :7].copy()
                lid[:, 6] = _yaw_filter(lid[:, 6])
                drop[fids[f]] = {'boxes_lidar': lid[d], 'score': boxes[s, f, :n, 7][d],
                                 'name': np.array([CLASS_NAMES[int(c) - 1] for c in boxes[s, f, :n, 8][d]]),
                                 'pose': poses[s, f].copy(), 'frame_id': fids[f], 'sequence_name': name}
            drops[name] = drop
        return tracks, drops


def track_sequences(boxes, counts, poses, num_frames=None, cfg=None, max_tracks=8192, max_entries=1 << 18):
    """The DetZero tracker on the device (csrc/tracker.cu).  boxes (S, F, K, 9) float32 CUDA lidar rows [x, y, z, dx, dy, dz, heading,
    score, label 1..3] (the gathered (F, K, 9) tensor of one sequence is S = 1), counts (S, F) rows per frame, poses (S, F, 4, 4)
    lidar -> world, num_frames (S) frames per sequence (default F).  max_tracks / max_entries: per-sequence capacity of track ids and
    of track entries (forward, reverse and output entries each); exceeding either raises.  Returns a TrackResult.
    Memory per sequence: a cached workspace of about 5.4 MB + 96 B per entry + 450 B per track id, and outputs of 84 B per entry +
    24 B per track id; at the defaults that is about 34 MB + 22 MB, so 3.6 GB for S = 64.  A track emits one entry per frame it
    is alive forward and one per frame before its start while its reverse track lives, so max_entries bounds the sum over frames of
    the live tracks."""
    c = _resolve_cfg(cfg)
    assert boxes.is_cuda and boxes.dtype == torch.float32 and boxes.shape[-1] == 9, (boxes.shape, boxes.dtype)
    if boxes.dim() == 3:
        boxes, counts, poses = boxes[None], torch.as_tensor(counts)[None], torch.as_tensor(poses)[None]
    S, F, K, _ = boxes.shape
    if K > 512:
        raise ValueError('at most 512 detections per frame (got K = %d)' % K)
    dev = boxes.device
    boxes = boxes.contiguous()
    counts = torch.as_tensor(counts).to(device=dev, dtype=torch.int32).reshape(S, F).contiguous()
    poses = torch.as_tensor(poses).to(device=dev, dtype=torch.float64).reshape(S, F, 4, 4).contiguous()
    nf = torch.full((S,), F, dtype=torch.int32) if num_frames is None else torch.as_tensor(num_frames)
    nf = nf.to(device=dev, dtype=torch.int32).reshape(S).contiguous()
    T, E = int(max_tracks), int(max_entries)
    i32 = dict(dtype=torch.int32, device=dev)
    trk = torch.zeros((S, T, 6), **i32)
    n_tracks = torch.zeros((S,), **i32)
    ent_box = torch.zeros((S, E, 9), dtype=torch.float64, device=dev)
    ent_score = torch.zeros((S, E), dtype=torch.float32, device=dev)
    ent_hit = torch.zeros((S, E), **i32)
    ent_frame = torch.zeros((S, E), **i32)
    kept = torch.zeros((S, F, K), dtype=torch.uint8, device=dev)
    overflow = torch.zeros((S,), **i32)
    if S:
        ws = ops.workspace(lib().dz_track_sequences_ws_bytes(S, F, K, T, E), dev, 'track')
        check(lib().dz_track_sequences(ops._p(boxes), ops._p(counts), ops._p(nf), ops._p(poses), S, F, K, _params(c), T, E,
                                       ops._p(trk), ops._p(n_tracks), ops._p(ent_box), ops._p(ent_score), ops._p(ent_hit),
                                       ops._p(ent_frame), ops._p(kept), ops._p(overflow), ops._p(ws), ws.numel(), ops._stream()),
              'track_sequences')
        ops._count(1)
    ov = overflow.cpu().numpy()
    if ov.any():
        s = int(np.flatnonzero(ov)[0])
        what = [n for b, n in ((1, 'track ids (max_tracks)'), (2, 'track entries (max_entries)'), (4, 'association edges'),
                               (8, 'assignment scratch'), (16, 'merge edges')) if ov[s] & b]
        raise RuntimeError('track_sequences: sequence %d exceeded the capacity of %s (max_tracks=%d, max_entries=%d)'
                           % (s, ', '.join(what), T, E))
    return TrackResult(boxes, counts, poses, nf, trk, n_tracks, ent_box, ent_score, ent_hit, ent_frame, kept.bool())


# ---------------------------------------------------------------------------------------------------------------------- ground truth
#: REFINING.IOU_THRESHOLDS of tracking/tools/cfgs/tk_model_cfgs/waymo_detzero_track.yaml (the assign-mode BEV IoU per class)
ASSIGN_IOU_THRESHOLDS = {'Vehicle': 0.3, 'Pedestrian': 0.1, 'Cyclist': 0.1}
#: match-rate cutoffs of TrackRecall (np.arange(0, 10) * 0.1, float64)
RECALL_CUTOFFS = np.arange(0, 10) * 0.1


class GroundTruth:
    """Ground truth of S sequences of up to F frames with up to G rows per frame (device tensors): box (S, F, G, 7) float32 lidar boxes
    (gt_boxes_lidar), world (S, F, G, 9) float64 (gt_boxes_global, velocity in columns 7:9), cls (S, F, G) int32 class 1..3 in
    CLASS_NAMES order or 0 for any other name (kept in the frame's row order, never matched), obj (S, F, G) the per-sequence object
    index (first appearance, -1 for a class-0 row), difficulty, num_points (num_points_in_gt), counts (S, F), num_frames (S), n_obj
    (S), poses (S, F, 4, 4) lidar -> world.  On the host: obj_ids[s][o] is object o's original obj_ids value, names[s] the per-frame
    name arrays and frame_ids[s][f] frame f's id (a string, as sequence_list_to_dict keys them)."""

    def __init__(self, box, world, cls, obj, difficulty, num_points, counts, num_frames, n_obj, poses, obj_ids, names, frame_ids):
        self.box, self.world, self.cls, self.obj = box, world, cls, obj
        self.difficulty, self.num_points, self.counts, self.num_frames, self.n_obj, self.poses = (difficulty, num_points, counts,
                                                                                                 num_frames, n_obj, poses)
        self.obj_ids, self.names, self.frame_ids = obj_ids, names, frame_ids

    def __len__(self):
        return self.box.shape[0]


def ground_truth_from_infos(infos, sequence_names, device='cuda'):
    """GroundTruth of the named sequences from the frame dicts of waymo_infos_<split>.pkl (info['annos'] with 'name', 'obj_ids',
    'gt_boxes_lidar', 'gt_boxes_global', 'difficulty', 'num_points_in_gt'; 'pose', 'sequence_name', 'sample_idx' or 'frame_id').
    Frames keep the order of ``infos`` within each sequence, so frame f of the table is frame f of a TrackResult of the same
    frames."""
    seqs = {}
    for info in infos:
        fid = str(info['sample_idx']) if 'sample_idx' in info else str(info['frame_id'])
        seqs.setdefault(info['sequence_name'], {})[fid] = info
    frames = [list(seqs[n].items()) for n in sequence_names]
    S = len(frames)
    F = max([len(fr) for fr in frames] + [1])
    G = max([len(i['annos']['name']) for fr in frames for _, i in fr] + [1])
    box = np.zeros((S, F, G, 7), np.float32)
    world = np.zeros((S, F, G, 9), np.float64)
    cls, obj, diff, npts = (np.zeros((S, F, G), np.int32) for _ in range(4))
    obj[:] = -1
    counts = np.zeros((S, F), np.int32)
    poses = np.tile(np.eye(4), (S, F, 1, 1))
    n_obj = np.zeros(S, np.int32)
    obj_ids, names, frame_ids = [], [], []
    for s, fr in enumerate(frames):
        index, ids = {}, []
        for f, (_, info) in enumerate(fr):
            a = info['annos']
            n = len(a['name'])
            counts[s, f] = n
            poses[s, f] = info['pose']
            if n == 0:
                continue
            box[s, f, :n] = np.asarray(a['gt_boxes_lidar'])[:, :7]
            gw = np.asarray(a['gt_boxes_global'], np.float64)
            world[s, f, :n, :gw.shape[1]] = gw
            diff[s, f, :n] = a['difficulty']
            npts[s, f, :n] = a['num_points_in_gt']
            for g in range(n):
                c = CLASS_NAMES.index(a['name'][g]) + 1 if a['name'][g] in CLASS_NAMES else 0
                cls[s, f, g] = c
                if c:
                    key = a['obj_ids'][g]
                    if key not in index:
                        index[key] = len(ids)
                        ids.append(key)
                    obj[s, f, g] = index[key]
        n_obj[s] = len(ids)
        obj_ids.append(ids)
        names.append([np.asarray(i['annos']['name']) for _, i in fr])
        frame_ids.append([fid for fid, _ in fr])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return GroundTruth(t(box), t(world), t(cls), t(obj), t(diff), t(npts), t(counts),
                       t(np.array([len(fr) for fr in frames], np.int32)), t(n_obj), t(poses), obj_ids, names, frame_ids)


class _Tracks:
    """the TrackResult fields the ground-truth scoring reads, for tracks given in the pickle form"""

    def __init__(self, trk, n_tracks, ent_box, ent_frame, poses, ids):
        self.trk, self.ent_box, self.ent_frame, self.poses, self.ids = trk, ent_box, ent_frame, poses, ids
        self.n_tracks = n_tracks


def _tracks_from_pickle(pred, gt, sequence_names):
    """{seq: {obj_id: {'boxes_global', 'name', 'sample_idx', ...}}} (the form TrackResult.to_reference writes) -> _Tracks, with the
    tracks of each sequence in dict order and their sample_idx mapped onto the ground truth's frames"""
    S = len(sequence_names)
    seqs = [pred[n] for n in sequence_names]
    T = max([len(p) for p in seqs] + [1])
    E = max([sum(len(t['name']) for t in p.values()) for p in seqs] + [1])
    trk = np.zeros((S, T, 6), np.int32)
    eb = np.zeros((S, E, 9), np.float64)
    ef = np.full((S, E), -1, np.int32)
    n_tracks, ids = np.zeros(S, np.int32), []
    for s, p in enumerate(seqs):
        fmap = {fid: f for f, fid in enumerate(gt.frame_ids[s])}
        off = 0
        ids.append(list(p.keys()))
        for k, (tid, t) in enumerate(p.items()):
            n = len(t['name'])
            cname = str(t['name'][0])
            if cname not in CLASS_NAMES:
                raise ValueError('track %r of sequence %r has class %r' % (tid, sequence_names[s], cname))
            fr = [fmap.get(str(x), -1) for x in t['sample_idx']]
            trk[s, k] = [k, CLASS_NAMES.index(cname) + 1, fr[0] if n else 0, n, 0, off]
            bx = np.asarray(t['boxes_global'], np.float64)
            eb[s, off:off + n, :bx.shape[1]] = bx[:, :9]
            ef[s, off:off + n] = fr
            off += n
        n_tracks[s] = len(p)
    dev = gt.box.device
    return _Tracks(torch.from_numpy(trk).to(dev), n_tracks, torch.from_numpy(eb).to(dev), torch.from_numpy(ef).to(dev), gt.poses, ids)


def _score(tracks, gt, thresholds, recall, iou_3d, max_pairs):
    """one launch of csrc/track_gt.cu -> (obj_rec (S, O, 5), trk_rec (S, T, 4), ent_iou (S, E)) device tensors"""
    S, F, G, _ = gt.box.shape
    if tracks.trk.shape[0] != S or tracks.poses.shape[1] != F:
        raise ValueError('tracks of %d sequences / %d frames against ground truth of %d / %d' % (tracks.trk.shape[0],
                                                                                              tracks.poses.shape[1], S, F))
    thr = [0.0, 0.0, 0.0]
    mask = 0
    for name, t in thresholds.items():
        if name not in CLASS_NAMES:
            raise ValueError('class %r is not one of %r' % (name, CLASS_NAMES))
        if not t > 0:
            raise ValueError('IoU thresholds must be positive (got %r for %r)' % (t, name))
        c = CLASS_NAMES.index(name) + 1
        thr[c - 1], mask = float(t), mask | (1 << c)
    dev = gt.box.device
    T, E = tracks.trk.shape[1], tracks.ent_box.shape[1]
    O = max(int(gt.n_obj.max()) if S else 0, 1)
    i32 = dict(dtype=torch.int32, device=dev)
    obj_rec = torch.zeros((S, O, 5), **i32)
    trk_rec = torch.zeros((S, T, 4), **i32)
    ent_iou = torch.zeros((S, E), dtype=torch.float32, device=dev)
    overflow = torch.zeros((S,), **i32)
    n_tracks = torch.as_tensor(np.asarray(tracks.n_tracks, np.int32)).to(dev)
    trk, ent_box = tracks.trk.contiguous(), tracks.ent_box.contiguous()
    ent_frame, poses = tracks.ent_frame.to(torch.int32).contiguous(), tracks.poses.to(torch.float64).contiguous()
    if S:
        ws = ops.workspace(lib().dz_track_gt_ws_bytes(S, F, O, T, E, int(max_pairs)), dev, 'track_gt')
        check(lib().dz_track_gt(ops._p(gt.box), ops._p(gt.world), ops._p(gt.cls), ops._p(gt.obj), ops._p(gt.difficulty),
                                ops._p(gt.num_points), ops._p(gt.counts), ops._p(gt.num_frames), ops._p(gt.n_obj), S, F, G, O,
                                ops._p(trk), ops._p(n_tracks), ops._p(ent_box), ops._p(ent_frame), ops._p(poses), T, E, darr(thr),
                                mask, int(recall), int(iou_3d), int(max_pairs), ops._p(obj_rec), ops._p(trk_rec), ops._p(ent_iou),
                                ops._p(overflow), ops._p(ws), ws.numel(), ops._stream()), 'track_gt')
        ops._count(1)
    ov = overflow.cpu().numpy()
    if ov.any():
        s = int(np.flatnonzero(ov)[0])
        what = [n for b, n in ((1, 'the pair table (max_pairs)'), (2, 'the assignment scratch')) if ov[s] & b]
        raise RuntimeError('track_gt: sequence %d exceeded the capacity of %s (max_pairs=%d)' % (s, ', '.join(what), max_pairs))
    return obj_rec, trk_rec, ent_iou


class AssignResult:
    """assign_track_target of S sequences (device tensors): obj_rec (S, O, 5) int32 per object [matched track row or -1, match
    count, trajectory length, L1/L2 bucket, class], trk_rec (S, T, 4) int32 per track row [matched object or -1, class, entry count,
    state (1 dynamic)], ent_iou (S, E) float32 per track entry the BEV IoU with the matched object in that frame (0 where the object
    is absent).  The state of an unmatched track is 0 here; to_reference keeps the tracker's state for it."""

    def __init__(self, obj_rec, trk_rec, ent_iou, track_result, gt):
        self.obj_rec, self.trk_rec, self.ent_iou = obj_rec, trk_rec, ent_iou
        self.track_result, self.gt = track_result, gt

    def matches(self, s=0):
        """(object index, track row) pairs of sequence s in object order (the reference's match rows)"""
        o = self.obj_rec[s, :int(self.gt.n_obj[s]), 0].cpu().numpy()
        return [(int(i), int(k)) for i, k in enumerate(o) if k >= 0]

    def to_reference(self, sequence_names, frame_ids=None):
        """{seq: {'label': {tk_id: {'track': ..., 'gt': ...}}, 'unlabel': {tk_id: {'track': ...}}}} as tracking/tools/run_track.py
        pickles it in assign mode: a labelled track gains 'iou' (float32 per box) and the 'state' of its object; 'gt' holds the
        object's gt_boxes_global, gt_boxes_lidar, name, obj_ids and sample_idx arrays.  Labels in match-row (object) order, the
        unlabelled tracks in track order."""
        frame_ids = self.gt.frame_ids if frame_ids is None else frame_ids
        tracks, _ = self.track_result.to_reference(sequence_names, frame_ids)
        trec, eiou = self.trk_rec.cpu().numpy(), self.ent_iou.cpu().numpy()
        gbox, gworld = self.gt.box.cpu().numpy(), self.gt.world.cpu().numpy()
        gobj, gcnt = self.gt.obj.cpu().numpy(), self.gt.counts.cpu().numpy()
        out = {}
        for s, name in enumerate(sequence_names):
            rows = self.track_result.tracks(s)
            fids = list(frame_ids[s])
            label, unlabel = {}, {}
            for o, k in self.matches(s):
                tid, off, cnt = int(rows[k][0]), int(rows[k][5]), int(rows[k][3])
                t = dict(tracks[name][tid])
                t['iou'] = eiou[s, off:off + cnt].copy()
                t['state'] = 'dynamic' if trec[s, k, 3] else 'static'
                fs, gs = np.nonzero(gobj[s, :len(fids)] == o)
                keep = gs < gcnt[s, fs]
                fs, gs = fs[keep], gs[keep]
                label[tid] = {'track': t, 'gt': {'gt_boxes_global': gworld[s, fs, gs].copy(), 'gt_boxes_lidar': gbox[s, fs, gs].copy(),
                                                 'name': np.array([self.gt.names[s][f][g] for f, g in zip(fs, gs)]),
                                                 'obj_ids': np.array([self.gt.obj_ids[s][o]] * len(fs)),
                                                 'sample_idx': np.array([str(fids[f]) for f in fs])}}
            for k in range(len(rows)):
                if trec[s, k, 0] < 0:
                    unlabel[int(rows[k][0])] = {'track': tracks[name][int(rows[k][0])]}
            out[name] = {'label': label, 'unlabel': unlabel}
        return out


def assign_track_target(track_result, gt, iou_thresholds=None, max_pairs=1 << 16):
    """target_assign.assign_track_target on the device (csrc/track_gt.cu) for every sequence of ``track_result`` against ``gt``
    (frame f of one is frame f of the other): per frame the class-masked BEV IoU of the ground-truth rows of the classes in
    ``iou_thresholds`` with the track boxes taken back to the lidar frame, per (object, track) the sum of the IoUs >= the class
    threshold over the object's trajectory length, and the GNN assignment on 1 - that similarity.  Returns an AssignResult.
    max_pairs: per-sequence capacity of (object, track) pairs with a positive IoU; exceeding it raises."""
    thr = dict(ASSIGN_IOU_THRESHOLDS if iou_thresholds is None else iou_thresholds)
    obj_rec, trk_rec, ent_iou = _score(track_result, gt, thr, False, False, max_pairs)
    return AssignResult(obj_rec, trk_rec, ent_iou, track_result, gt)


def tracklet_recall(track_result, gt, class_names=CLASS_NAMES, iou_threshold=(0.7, 0.5, 0.5), method='3d',
                    difficultys=('l1', 'l2'), sequence_names=None, max_pairs=1 << 16):
    """TrackRecall.get_tracklet_recall (tracking/detzero_track/utils/track_recall.py) over every sequence of the call: per sequence
    the class-masked 3-D (method '3d') or BEV ('bev') IoU, per (object, track) the sum of the same-frame IoUs over the object's
    trajectory length and the count of IoUs >= the class threshold, the GNN assignment (csrc/track_gt.cu), then on the host from one
    copy of the per-object and per-track records: {difficulty: {class: {'precisions', 'recalls', 'tp', 'fp', 'pred_nums', 'cutoffs',
    'gt_nums'}}, 'iou_thresholds': {class: threshold}, 'method': method}.
    ``track_result`` is a TrackResult or predictions in the pickle form {seq: {obj_id: {'boxes_global', 'name', 'sample_idx'}}}
    (TrackResult.to_reference writes it), scored against the sequences ``sequence_names`` (default: its keys in order) of ``gt``.
    A match rate is the float32 quotient match count / trajectory length, compared with the float64 cutoffs (numpy >= 2 arithmetic
    of the reference).  Where the reference raises (a difficulty and class with ground truth but no matched trajectory has no
    match rates), tp is 0."""
    if tuple(difficultys) != ('l1', 'l2'):
        raise ValueError("difficultys must be ('l1', 'l2') (got %r)" % (difficultys,))
    if method not in ('3d', 'bev'):
        raise ValueError('method must be 3d or bev (got %r)' % (method,))
    class_names = list(class_names)
    if len(class_names) != len(iou_threshold):
        raise ValueError('one IoU threshold per class')
    thr = dict(zip(class_names, iou_threshold))
    if isinstance(track_result, dict):
        names = list(track_result.keys()) if sequence_names is None else list(sequence_names)
        tracks = _tracks_from_pickle(track_result, gt, names)
    else:
        tracks = _Tracks(track_result.trk, track_result.n_tracks, track_result.ent_box, track_result.ent_frame, gt.poses, None)
    obj_rec, trk_rec, _ = _score(tracks, gt, thr, True, method == '3d', max_pairs)
    orec, trec = obj_rec.cpu().numpy(), trk_rec.cpu().numpy()
    rates = {d: {c: [] for c in class_names} for d in difficultys}
    gt_nums = {d: {c: 0 for c in class_names} for d in difficultys}
    pred_nums = {d: {c: 0 for c in class_names} for d in difficultys}
    bucket = {1: 'l1', 2: 'l2'}
    for s in range(len(gt)):
        for k, cnt, ln, b, c in orec[s, :int(gt.n_obj[s])]:
            if ln == 0:
                continue
            d, name = bucket[int(b)], CLASS_NAMES[c - 1]
            gt_nums[d][name] += 1
            if k >= 0:
                rates[d][name].append(np.float32(cnt) / np.float32(ln))
                pred_nums[d][name] += 1
        for o, c, n, _ in trec[s, :int(tracks.n_tracks[s])]:
            if o < 0:
                name = CLASS_NAMES[c - 1]
                if name not in class_names:
                    raise ValueError('a track of class %r is not in class_names' % name)
                for d in difficultys:
                    pred_nums[d][name] += 1
    out = {}
    for d in difficultys:
        out[d] = {}
        for c in class_names:
            r = np.array(rates[d][c], np.float32)
            g, p = gt_nums[d][c], pred_nums[d][c]
            res = {'precisions': [], 'recalls': [], 'tp': [], 'fp': [], 'pred_nums': [], 'cutoffs': [], 'gt_nums': []}
            for cut in RECALL_CUTOFFS:
                tp = int(np.count_nonzero(r >= cut)) if g > 0 else 0
                fp = p - tp
                res['precisions'].append(tp / (tp + fp + 1e-9))
                res['recalls'].append(tp / (g + 1e-9))
                res['tp'].append(tp)
                res['fp'].append(fp)
                res['pred_nums'].append(p)
                res['cutoffs'].append(float(cut))
                res['gt_nums'].append(g)
            out[d][c] = res
    out['iou_thresholds'] = thr
    out['method'] = method
    return out

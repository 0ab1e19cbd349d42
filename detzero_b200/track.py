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

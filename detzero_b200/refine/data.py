"""Refiner inputs on the device: crop each track's points from its frames, sample and encode the PRM / GRM / CRM features, and map
refined boxes back to each frame (csrc/refine_data.cu, include/detzero_b200.h dz_refine_inputs / dz_refine_revert).

Replaces the eval branch of WaymoPositionDataset / WaymoGeometryDataset / WaymoConfidenceDataset.extract_track_feature and
revert_to_each_frame (refining/detzero_refine/datasets/waymo/), together with the per-object crop of
daemon/prepare_object_data.py:241-327.  Each builder returns the dict the modules of detzero_b200.refine consume, with the
reference's keys, shapes and float32 dtype.  Sampling is keyed on (seed, track_uid) and deterministic; see csrc/refine_data.cu for
that function and the other deliberate deviations (float64 geometry, per-track GRM query count, the crop's coordinates).
``combine_frames`` puts the refined tracks of a sequence together into per-frame result rows (csrc/combine.cu), replacing
daemon/combine_output.py's convert_frame_format and combine_det.
"""
import zlib

import numpy as np
import torch

from .. import ops
from .._lib import check, lib

PRM, CRM, GRM = 0, 1, 2
CLASS_MAP = {'Vehicle': 1, 'Pedestrian': 2, 'Cyclist': 3}
#: the ENCODING lists of the shipped configs (refining/tools/cfgs/ref_{dataset,model}_cfgs); anything else is an error
P2CO = ['xyz', 'intensity', 'p2co', 'score']
P2CO_CLASS = P2CO + ['class']
P2S = ['xyz', 'intensity', 'p2s', 'score']


def _cfg(cfg, defaults):
    out = dict(defaults)
    if cfg is not None:
        out.update({k: cfg[k] for k in cfg.keys()})
    return out


def prm_data_cfg():
    """waymo_prm_dataset.yaml (+ the daemon's crop settings, prepare_object_data.py:21)"""
    return {'ENCODING': list(P2CO), 'QUERY_NUM': 200, 'QUERY_POINTS_NUM': 256, 'MEMORY_POINTS_NUM': 48, 'ENLARGE_SCALE': 1.1,
            'CROP_ON_BEV': False}


def crm_data_cfg():
    """waymo_crm_dataset.yaml"""
    return {'ENCODING': list(P2CO), 'QUERY_NUM': 200, 'QUERY_POINTS_NUM': 256, 'ENLARGE_SCALE': 1.1, 'CROP_ON_BEV': False}


def grm_data_cfg():
    """waymo_grm_dataset.yaml"""
    return {'ENCODING': list(P2S), 'QUERY_NUM': 3, 'QUERY_POINTS_NUM': 256, 'MEMORY_POINTS_NUM': 4096, 'ENLARGE_SCALE': 1.1,
            'CROP_ON_BEV': False}


class TrackBatch:
    """Device track tables of B tracks with up to L box slots (L = QUERY_NUM of PRM / CRM, 200):
    boxes (B, L, 7) float64 world [x, y, z, dx, dy, dz, heading], frame_of_box (B, L) int32 (index into the frames / poses),
    scores (B, L) float32, box_num (B) int32 in 1..L, cls (B) int32 (1 Vehicle, 2 Pedestrian, 3 Cyclist), track_uid (B) int64
    (the sampling key: a track's inputs depend on (seed, track_uid) only)."""

    def __init__(self, boxes, frame_of_box, scores, box_num, cls, track_uid, device='cuda'):
        box_num = torch.as_tensor(np.asarray(box_num) if not torch.is_tensor(box_num) else box_num).to(torch.int32)
        B, L = int(box_num.shape[0]), int(np.shape(boxes)[1])
        bn = box_num.cpu()
        if B and (int(bn.min()) < 1 or int(bn.max()) > L):
            raise ValueError('box_num must lie in 1..%d' % L)
        self.boxes = torch.as_tensor(boxes, dtype=torch.float64).reshape(B, L, 7).to(device).contiguous()
        self.frame_of_box = torch.as_tensor(frame_of_box).to(device=device, dtype=torch.int32).reshape(B, L).contiguous()
        self.scores = torch.as_tensor(scores).to(device=device, dtype=torch.float32).reshape(B, L).contiguous()
        self.box_num = bn.to(device)
        self.cls = torch.as_tensor(cls).to(device=device, dtype=torch.int32).reshape(B).contiguous()
        self.track_uid = torch.as_tensor(track_uid).to(device=device, dtype=torch.int64).reshape(B).contiguous()
        self.max_box_num = int(bn.max()) if B else 0

    def __len__(self):
        return self.box_num.shape[0]

    @property
    def L(self):
        return self.boxes.shape[1]

    def select(self, idx):
        """the tracks idx (a slice or an index list) as a TrackBatch"""
        return TrackBatch(self.boxes[idx], self.frame_of_box[idx], self.scores[idx], self.box_num[idx], self.cls[idx],
                          self.track_uid[idx], self.boxes.device)


def _frames_args(frames, frame_offsets, poses):
    assert frames.is_cuda and frames.dtype == torch.float32 and frames.dim() == 2 and frames.shape[1] >= 5 and frames.stride(1) == 1
    off_host = np.asarray(frame_offsets.cpu() if torch.is_tensor(frame_offsets) else frame_offsets, np.int64)
    F = len(off_host) - 1
    if F < 1 or off_host[0] != 0 or np.any(np.diff(off_host) < 0) or off_host[-1] > frames.shape[0]:
        raise ValueError('frame_offsets must be F + 1 non-decreasing row offsets into frames')
    off = torch.from_numpy(off_host.astype(np.int32)).to(frames.device)
    poses = poses.to(device=frames.device, dtype=torch.float64).contiguous()
    assert poses.shape == (F, 4, 4), (poses.shape, F)
    return off, F, int(np.diff(off_host).max()), poses


def _build(kind, frames, frame_offsets, poses, tracks, cfg, seed, crop, return_selection):
    enc = list(cfg['ENCODING'])
    if kind == GRM and enc != P2S or kind != GRM and enc not in (P2CO, P2CO_CLASS) or kind == CRM and enc != P2CO:
        raise ValueError('unsupported ENCODING %r (the shipped lists only)' % (enc,))
    with_class = enc == P2CO_CLASS
    off, F, max_pts, poses = _frames_args(frames, frame_offsets, poses)
    dev = frames.device
    B, L = len(tracks), tracks.L
    if kind != GRM and int(cfg['QUERY_NUM']) != L:
        raise ValueError('QUERY_NUM %d != the track tables\' %d box slots' % (cfg['QUERY_NUM'], L))
    kq = int(cfg['QUERY_POINTS_NUM'])
    km = int(cfg.get('MEMORY_POINTS_NUM', 0)) if kind != CRM else 0
    nq = int(cfg['QUERY_NUM']) if kind == GRM else 1
    q_out = min(nq, tracks.max_box_num) if kind == GRM else 0
    C = 4 if kind == GRM else 32 + (3 if with_class else 0)
    f32 = dict(dtype=torch.float32, device=dev)
    if kind == GRM:
        q = torch.empty((B, q_out, kq, 4), **f32)
        m = torch.empty((B, km, 11), **f32)
        traj = torch.empty((B, L, 7), **f32)
        box_f = torch.empty((B, q_out, 7), **f32)
        track_f = None
        qn = torch.empty((B,), dtype=torch.int32, device=dev)
        nsel = nq * kq + km
    else:
        q = torch.empty((B, L, kq, C), **f32)
        m = torch.empty((B, L, km, C), **f32) if kind == PRM else None
        traj = torch.empty((B, L, 7), **f32) if kind == PRM else None
        box_f = torch.empty((B, L), **f32)
        track_f = torch.empty((B, 7), **f32) if kind == PRM else None
        qn = None
        nsel = L * (kq + km)
    counts = torch.empty((B, L), dtype=torch.int32, device=dev) if return_selection else None
    sel = torch.full((B, nsel), -1, dtype=torch.int32, device=dev) if return_selection else None
    if B:
        ws = ops.workspace(lib().dz_refine_inputs_ws_bytes(kind, B, L, max_pts, kq, km, nq), dev, 'refine_data')
        check(lib().dz_refine_inputs(kind, ops._p(frames), frames.stride(0), ops._p(off), F, max_pts, ops._p(poses),
                                     ops._p(tracks.boxes), ops._p(tracks.frame_of_box), ops._p(tracks.scores), ops._p(tracks.box_num),
                                     ops._p(tracks.cls), ops._p(tracks.track_uid), B, L, kq, km, nq, q_out, int(with_class),
                                     float(cfg.get('ENLARGE_SCALE', 1.1)), int(bool(cfg.get('CROP_ON_BEV', False))), int(bool(crop)),
                                     int(seed) & ((1 << 64) - 1), ops._p(q), ops._p(m), ops._p(traj), ops._p(box_f), ops._p(track_f),
                                     ops._p(qn), ops._p(counts), ops._p(sel), ops._p(ws), ws.numel(), ops._stream()),
              'refine_inputs')
        ops._count(7)
    if kind == PRM:
        out = {'pos_query_points': q, 'pos_memory_points': m, 'pos_trajectory': traj, 'padding_mask': box_f,
               'pos_init_box': track_f, 'box_num': tracks.box_num}
    elif kind == CRM:
        out = {'conf_points': q, 'conf_score': box_f, 'box_num': tracks.box_num}
    else:
        out = {'geo_query_points': q, 'geo_query_boxes': box_f, 'geo_memory_points': m, 'geo_query_num': qn, 'geo_trajectory': traj}
    if return_selection:
        out['crop_counts'], out['selection'] = counts, sel
    return out


def position_inputs(frames, frame_offsets, poses, tracks, cfg=None, seed=0, crop=True, return_selection=False):
    """PRM inputs (WaymoPositionDataset.extract_track_feature, eval) of every track.
    frames: (N, >=5) CUDA float32 collated rows [b, x, y, z, tanh(i), ...] (io.prepare_points / FramePipeline), lidar frame;
    frame_offsets (F + 1) row offsets (host or device); poses (F, 4, 4) float64 lidar -> world; tracks: TrackBatch.
    crop=False: every point of a box's frame is its point set (tracks_from_object_infos).  return_selection adds 'crop_counts' (B, L)
    and 'selection' (B, L * (kq + km)): per box the sorted kept ranks of the query then the memory sample (-1 unused)."""
    return _build(PRM, frames, frame_offsets, poses, tracks, _cfg(cfg, prm_data_cfg()), seed, crop, return_selection)


def confidence_inputs(frames, frame_offsets, poses, tracks, cfg=None, seed=0, crop=True, return_selection=False):
    """CRM inputs (WaymoConfidenceDataset.extract_track_feature, eval); arguments as position_inputs ('selection' (B, L * kq))"""
    return _build(CRM, frames, frame_offsets, poses, tracks, _cfg(cfg, crm_data_cfg()), seed, crop, return_selection)


def geometry_inputs(frames, frame_offsets, poses, tracks, cfg=None, seed=0, crop=True, return_selection=False):
    """GRM inputs (WaymoGeometryDataset.extract_track_feature, eval), geo_query_points / boxes padded to the batch's largest
    geo_query_num (dataset.py:239-256); 'geo_trajectory' is the world trajectory.  'selection' (B, nq * kq + km): the kept ranks of
    each query box, then of the memory sample over the concatenation of every box's points."""
    return _build(GRM, frames, frame_offsets, poses, tracks, _cfg(cfg, grm_data_cfg()), seed, crop, return_selection)


def _revert(kind, pred, poses, tracks):
    B, L = len(tracks), tracks.L
    dev = tracks.boxes.device
    pred = pred.to(device=dev, dtype=torch.float32).contiguous()
    assert pred.shape == ((B, L, 7) if kind == PRM else (B, 7)), pred.shape
    poses = poses.to(device=dev, dtype=torch.float64).contiguous()
    lidar = torch.empty((B, L, 7), dtype=torch.float64, device=dev)
    world = torch.empty((B, L, 7), dtype=torch.float64, device=dev)
    if B:
        check(lib().dz_refine_revert(kind, ops._p(pred), ops._p(poses), poses.shape[0], ops._p(tracks.boxes), ops._p(tracks.frame_of_box),
                                     ops._p(tracks.box_num), B, L, ops._p(lidar), ops._p(world), ops._stream()), 'refine_revert')
        ops._count(1)
    return lidar, world


def revert_position_boxes(pred_boxes, poses, tracks):
    """WaymoPositionDataset.revert_to_each_frame: PRM boxes (B, L, 7) in each track's init-box frame -> (lidar, world), each
    (B, L, 7) float64, rows past box_num zero"""
    return _revert(PRM, pred_boxes, poses, tracks)


def revert_geometry_boxes(pred_boxes, poses, tracks):
    """WaymoGeometryDataset.revert_to_each_frame: the GRM size (B, 7) written into every world box -> (lidar, world) (B, L, 7)"""
    return _revert(GRM, pred_boxes, poses, tracks)


def combine_frames(prm_lidar, grm_pred, scores, frame_of_box, box_num, cls, track_id, num_frames, drop=None, max_rows=1024):
    """convert_frame_format + combine_det (daemon/combine_output.py) on the device (csrc/combine.cu): the refined tracks of one
    sequence -> per-frame result rows.  Tables of the B tracks in output order (combine_final's: class by class, ids ascending):
    prm_lidar (B, L, 7) f64 (revert_position_boxes' lidar boxes), grm_pred (B, 7) (the GRM prediction; only its size is used),
    scores (B, L) f32 (the CRM pred_score, or the tracker's per-box score), frame_of_box (B, L) sequence frame indices 0..num_frames-1
    (a caller whose frame_of_box is not one, e.g. after tracks_from_object_infos, passes the sequence frame index here), box_num (B),
    cls (B) 1..3, track_id (B) in 0..2**31-1, unique.  drop: None, or the tracker's dropped detections of the sequence as
    (det (>= num_frames, K, 9) f32 gathered rows, counts, kept (.., K) bool), e.g. (res.boxes[s], res.counts[s], res.kept[s]) of a
    TrackResult.
    Returns rows (F, R, 9) f32 [x, y, z, dx, dy, dz, heading, score, label], obj_id (F, R) int32 (-1: a dropped detection) and
    count (F) int32, R = max_rows; rows past count[f] are zero with obj_id -1.  A frame's rows are its track boxes (PRM box with
    the GRM size, by track then box order), then its dropped detections in input order with det_drop's heading wrap.  A frame
    without a track box has no row at all.  Raises if a frame needs more than max_rows rows.
    Deviations from combine_final: one call combines every class given (the reference writes one accumulating file per class), and a
    frame with tracks but no detections has no dropped row (combine_det raises KeyError there)."""
    dev = prm_lidar.device
    B, L = int(prm_lidar.shape[0]), int(prm_lidar.shape[1])
    F, R = int(num_frames), int(max_rows)
    if F < 1 or R < 1:
        raise ValueError('num_frames and max_rows must be positive')
    i32 = dict(dtype=torch.int32, device=dev)
    prm = prm_lidar.to(dtype=torch.float64).contiguous()
    assert prm.shape == (B, L, 7), prm.shape
    grm = torch.as_tensor(grm_pred).to(device=dev, dtype=torch.float32).reshape(B, 7).contiguous()
    sc = torch.as_tensor(scores).to(device=dev, dtype=torch.float32).reshape(B, L).contiguous()
    fob = torch.as_tensor(frame_of_box).to(**i32).reshape(B, L).contiguous()
    bn = torch.as_tensor(box_num).to(**i32).reshape(B).contiguous()
    cl = torch.as_tensor(cls).to(**i32).reshape(B).contiguous()
    tid = torch.as_tensor(track_id).to(device=dev, dtype=torch.int64).reshape(B)
    if B:
        lo, hi = torch.stack([tid.min(), tid.max()]).tolist()
        if lo < 0 or hi >= 1 << 31:
            raise ValueError('track ids must lie in 0..2**31-1 (got %d..%d)' % (lo, hi))
    tid = tid.to(torch.int32).contiguous()
    det = cnt = kept = None
    K = 0
    if drop is not None:
        det, cnt, kept = drop
        assert det.dim() == 3 and det.shape[0] >= F and det.shape[2] == 9, det.shape
        K = int(det.shape[1])
        det = det[:F].to(device=dev, dtype=torch.float32).contiguous()
        cnt = torch.as_tensor(cnt)[:F].to(**i32).contiguous()
        kept = torch.as_tensor(kept)[:F].to(device=dev, dtype=torch.uint8).reshape(F, K).contiguous()
    rows = torch.zeros((F, R, 9), dtype=torch.float32, device=dev)
    obj_id = torch.full((F, R), -1, **i32)
    count = torch.empty((F,), **i32)
    overflow = torch.zeros((1,), **i32)
    ws = ops.workspace(lib().dz_combine_frames_ws_bytes(B, L, F), dev, 'combine')
    check(lib().dz_combine_frames(ops._p(prm), ops._p(grm), ops._p(sc), ops._p(fob), ops._p(bn), ops._p(cl), ops._p(tid), B, L,
                                  ops._p(det), ops._p(cnt), ops._p(kept), K, F, R, ops._p(rows), ops._p(obj_id), ops._p(count),
                                  ops._p(overflow), ops._p(ws), ws.numel(), ops._stream()), 'combine_frames')
    ops._count(3)
    ov = int(overflow.item())
    if ov & 2:
        raise ValueError('combine_frames: a frame_of_box entry lies outside 0..%d' % (F - 1))
    if ov & 1:
        raise RuntimeError('combine_frames: a frame needs more than max_rows=%d rows' % R)
    return rows, obj_id, count


def tracks_from_object_infos(obj_infos, L=200, track_uid=None, device='cuda'):
    """Host packer for the per-object pickles of daemon/prepare_object_data.py (a list of per-object dicts with 'boxes_global',
    'score', 'pose', 'pts' (global float64 [x, y, z, tanh(i)] per box) and 'name').  Each box's points go back to its lidar frame in
    float64 and every box becomes its own frame, so the builders run with crop=False.  track_uid defaults to crc32 of the obj_id.
    Returns (frames, frame_offsets, poses, TrackBatch)."""
    B = len(obj_infos)
    boxes = np.zeros((B, L, 7))
    fob = np.zeros((B, L), np.int32)
    scores = np.zeros((B, L), np.float32)
    box_num = np.zeros(B, np.int32)
    cls = np.zeros(B, np.int32)
    rows, offsets, poses = [], [0], []
    for b, info in enumerate(obj_infos):
        n = len(info['boxes_global'])
        if not 1 <= n <= L:
            raise ValueError('track %d has %d boxes (1..%d supported)' % (b, n, L))
        box_num[b] = n
        boxes[b, :n] = np.asarray(info['boxes_global'], np.float64)[:, :7]
        scores[b, :n] = np.asarray(info['score'], np.float32)
        cls[b] = CLASS_MAP[info['name']]
        for j in range(n):
            P = np.asarray(info['pose'][j], np.float64)
            p = np.asarray(info['pts'][j], np.float64).reshape(-1, 4)
            loc = (p[:, :3] - P[:3, 3]) @ P[:3, :3]                     # inverse of the rigid pose
            r = np.zeros((len(p), 6), np.float32)
            r[:, 1:4], r[:, 4] = loc, p[:, 3]
            rows.append(r)
            fob[b, j] = len(poses)
            poses.append(P)
            offsets.append(offsets[-1] + len(p))
    if track_uid is None:
        track_uid = [zlib.crc32(str(info.get('obj_id', b)).encode()) for b, info in enumerate(obj_infos)]
    frames = torch.from_numpy(np.concatenate(rows, 0) if rows else np.zeros((0, 6), np.float32)).to(device)
    return (frames, np.asarray(offsets, np.int64), torch.from_numpy(np.stack(poses)).to(device),
            TrackBatch(boxes, fob, scores, box_num, cls, np.asarray(track_uid, np.int64), device))

"""Waymo detection AP and APH per object type, difficulty level and range on the device (csrc/det_eval.cu), as DetZero's evaluator
reports them (evaluator/detzero_eval.py -> WaymoDetectionMetricsEstimator.waymo_evaluation,
detection/detzero_det/datasets/waymo/waymo_eval_detection.py), without TensorFlow or the Waymo metric library.

  * ``detection_metrics`` -- padded per-frame device tables in, the int64 records (16 shards x 2 levels x 101 score cutoffs x
    [TP, FP, FN, TPH]) and the AP dict out.
  * ``WaymoDetectionMetricsEstimator().waymo_evaluation`` -- the reference's entry point on its frame dicts.
  * ``evaluate_offboard`` -- the final boxes of offboard.refine_sequence against a track.GroundTruth, prepared with torch
    elementwise ops on the device.

The metric (stated in full in csrc/det_eval.cu): per frame, shard and cutoff the shard's ground truth is matched to the active
predictions of its type by the maximum IoU sum over pairs at or above the type's IoU threshold; TP / FP / FN / TPH are counted per
level; AP is the area under the precision envelope of the 101 (recall, precision) points, APH the same with TPH in place of TP
in the numerators of precision and recall.
Compatibility with the official Waymo metric is not verified.  Points where the definition is this project's choice, not pinned
by the reference: a RANGE shard matches its ground truth against predictions of every range and counts an FP in the prediction's
own range only when it is matched in none of the type's range matchings; IoU is DetZero's boxes_iou3d_gpu (3d) or its rotated BEV
IoU (bev), not Waymo's; ties in the matching follow the first minimum of the Hungarian's column scan; no interpolation between
distant recall points.

Tracking mode (evaluator/detzero_eval.py --tracking -> WaymoTrackingMetricsEstimator, evaluator/waymo_eval_tracking.py): MOTA, MOTP,
MISS, MISMATCH and FP per object type, level and range on the device (csrc/track_eval.cu, which states the CLEAR-MOT definition in
full): ``tracking_metrics`` on padded per-sequence device tables, ``mot_dict`` on the host, ``WaymoTrackingMetricsEstimator`` on
the reference's frame dicts, ``evaluate_tracks`` on track.track_sequences results and ``evaluate_offboard_tracking`` on
offboard.refine_sequence results.  Per (sequence, type, cutoff) a chain keeps last frame's still-valid pairs, matches the rest by
the maximum IoU sum, and counts a mismatch when an object's last matched id changes; RANGE splits the counts of that one chain by
the ground-truth box's range (the prediction's for an FP), unlike the detection RANGE above.  Compatibility with the official Waymo
tracking metric is not verified."""
import numpy as np
import torch

from . import ops
from ._lib import check, lib
from .track import CLASS_NAMES

#: the reference's WAYMO_CLASSES: name -> Waymo type index (type 3 is Waymo's SIGN)
WAYMO_CLASSES = ['unknown', 'Vehicle', 'Pedestrian', 'Truck', 'Cyclist']
TYPE_NAMES = ['VEHICLE', 'PEDESTRIAN', 'SIGN', 'CYCLIST']
RANGE_NAMES = ['[0, 30)', '[30, 50)', '[50, +inf)']
CONFIG_TYPES = ('object', 'range', '3d', 'bev')
NUM_CUTOFFS = 101
_FIXED = 2.0 ** 32


def _config(config_type):
    for c in config_type:
        if c not in CONFIG_TYPES:
            raise ValueError('unknown config type %r (supported: %s)' % (c, ', '.join(CONFIG_TYPES)))
    breakdowns = tuple(b for b in ('object', 'range') if b in config_type)
    return breakdowns, ('bev' if 'bev' in config_type and '3d' not in config_type else '3d')


def average_precision(tp, fp, fn, tph=None):
    """area under the precision envelope of the (recall, precision) points of the cutoffs, in recall order from recall 0: the sum of
    (r_i - r_{i-1}) * max{p_j : r_j >= r_i}, p = TP / (TP + FP) (0 where nothing is active), r = TP / (TP + FN) (0 where nothing
    counts).  With tph (APH) the heading-weighted TP replaces TP in both numerators."""
    tp, fp, fn = (np.asarray(a, np.float64) for a in (tp, fp, fn))
    num = tp if tph is None else np.asarray(tph, np.float64)
    with np.errstate(invalid='ignore', divide='ignore'):
        p = np.where(tp + fp > 0, num / (tp + fp), 0.0)
        r = np.where(tp + fn > 0, num / (tp + fn), 0.0)
    order = np.argsort(r, kind='stable')
    rs, env = r[order], np.maximum.accumulate(p[order][::-1])[::-1]
    ap, prev = 0.0, 0.0
    for i in range(len(rs)):
        ap += (rs[i] - prev) * env[i]
        prev = rs[i]
    return float(ap)


def ap_dict(records, breakdowns=('object',)):
    """{'OBJECT_TYPE_TYPE_VEHICLE_LEVEL_1/AP': [ap], ..., 'RANGE_TYPE_CYCLIST_[50, +inf)_LEVEL_2/APH': [aph]} from the records
    (16, 2, 101, 4) of the breakdowns; SIGN keys are always present.  A shard without counting ground truth gets 0."""
    rec = np.asarray(records)
    shards = []
    if 'object' in breakdowns:
        shards += [(t, 'OBJECT_TYPE_TYPE_%s' % TYPE_NAMES[t]) for t in range(4)]
    if 'range' in breakdowns:
        shards += [(4 + 3 * t + r, 'RANGE_TYPE_%s_%s' % (TYPE_NAMES[t], RANGE_NAMES[r])) for t in range(4) for r in range(3)]
    out = {}
    for s, name in shards:
        for lvl in (0, 1):
            tp, fp, fn, tph = (rec[s, lvl, :, i].astype(np.float64) for i in range(4))
            if tp[0] + fn[0] == 0:
                ap = aph = 0.0
            else:
                ap, aph = average_precision(tp, fp, fn), average_precision(tp, fp, fn, tph / _FIXED)
            out['%s_LEVEL_%d/AP' % (name, lvl + 1)] = [ap]
            out['%s_LEVEL_%d/APH' % (name, lvl + 1)] = [aph]
    return out


def detection_metrics(pred, pred_cnt, gt_box, gt_type, gt_level, gt_cnt, box_type='3d', breakdowns=('object',), max_pairs=1 << 14,
                      frame_chunk=None):
    """Records and AP dict of NF frames on the device (csrc/det_eval.cu).  pred (NF, R, 9) f32 CUDA [x, y, z, dx, dy, dz, heading,
    score, Waymo type], pred_cnt (NF) rows per frame; gt_box (NF, G, 7) f32, gt_type (NF, G) Waymo type, gt_level (NF, G) 1 or 2,
    gt_cnt (NF).  Rows of a type outside 1..4 are ignored.  box_type '3d' or 'bev'; breakdowns from 'object', 'range'.
    max_pairs: capacity of valid (IoU >= threshold) pairs per frame; exceeding it raises.  frame_chunk: frames per launch (bounds
    the workspace; records add up over chunks, so it does not change the result).  Returns (records (16, 2, 101, 4) int64 numpy
    [shard][level][cutoff][TP, FP, FN, TPH in 2^-32 units], ap dict); one device-to-host copy."""
    if box_type not in ('3d', 'bev'):
        raise ValueError('box_type must be 3d or bev (got %r)' % (box_type,))
    for b in breakdowns:
        if b not in ('object', 'range'):
            raise ValueError('unknown breakdown %r' % (b,))
    assert pred.is_cuda and pred.dtype == torch.float32 and pred.dim() == 3 and pred.shape[2] == 9, (pred.shape, pred.dtype)
    assert gt_box.is_cuda and gt_box.dtype == torch.float32 and gt_box.dim() == 3 and gt_box.shape[2] == 7, (gt_box.shape, gt_box.dtype)
    NF, dev = pred.shape[0], pred.device
    if gt_box.shape[0] != NF:
        raise ValueError('%d prediction frames against %d ground-truth frames' % (NF, gt_box.shape[0]))
    i32 = lambda t: torch.as_tensor(t).to(device=dev, dtype=torch.int32).contiguous()
    pred_cnt, gt_type, gt_level, gt_cnt = i32(pred_cnt).reshape(NF), i32(gt_type), i32(gt_level), i32(gt_cnt).reshape(NF)
    if pred.shape[1] == 0:
        pred, pred_cnt = torch.zeros((NF, 1, 9), dtype=torch.float32, device=dev), torch.zeros_like(pred_cnt)
    if gt_box.shape[1] == 0:
        gt_box, gt_cnt = torch.zeros((NF, 1, 7), dtype=torch.float32, device=dev), torch.zeros_like(gt_cnt)
        gt_type = gt_level = torch.zeros((NF, 1), dtype=torch.int32, device=dev)
    pred, gt_box = pred.contiguous(), gt_box.contiguous()
    R, G = pred.shape[1], gt_box.shape[1]
    if tuple(gt_type.shape) != (NF, G) or tuple(gt_level.shape) != (NF, G):
        raise ValueError('gt_type / gt_level must be (NF, G) = (%d, %d)' % (NF, G))
    records = torch.zeros((16, 2, NUM_CUTOFFS, 4), dtype=torch.int64, device=dev)
    overflow = torch.zeros((1,), dtype=torch.int32, device=dev)
    mask = sum(1 << i for i, b in enumerate(('object', 'range')) if b in breakdowns)
    chunk = NF if frame_chunk is None else max(int(frame_chunk), 1)
    if NF and mask:
        ws = ops.workspace(lib().dz_det_eval_ws_bytes(min(chunk, NF), R, G, int(max_pairs)), dev, 'det_eval')
        for f0 in range(0, NF, chunk):
            f1 = min(f0 + chunk, NF)
            check(lib().dz_det_eval(ops._p(pred[f0:f1]), ops._p(pred_cnt[f0:f1]), ops._p(gt_box[f0:f1]), ops._p(gt_type[f0:f1]),
                                    ops._p(gt_level[f0:f1]), ops._p(gt_cnt[f0:f1]), f1 - f0, R, G, int(box_type == 'bev'), mask,
                                    int(max_pairs), ops._p(records), ops._p(overflow), ops._p(ws), ws.numel(), ops._stream()),
                  'det_eval')
            ops._count(1)
    out = torch.cat([records.reshape(-1), overflow.long()]).cpu().numpy()
    rec, ov = out[:-1].reshape(16, 2, NUM_CUTOFFS, 4), int(out[-1])
    if ov:
        what = [n for b, n in ((1, 'valid pairs per frame (max_pairs=%d)' % max_pairs), (2, 'the assignment scratch')) if ov & b]
        raise RuntimeError('det_eval: a frame exceeded the capacity of %s' % ', '.join(what))
    return rec, ap_dict(rec, breakdowns)


def _limit_period(val, offset=0.5, period=np.pi):
    return val - np.floor(val / period + offset) * period


def _fakelidar_to_lidar(b):
    """boxes3d_kitti_fakelidar_to_lidar of generate_waymo_type_results (on a copy)"""
    b = np.array(b)
    w, l, h, r = b[:, 3:4], b[:, 4:5], b[:, 5:6], b[:, 6:7]
    b[:, 2] += h[:, 0] / 2
    return np.concatenate([b[:, 0:3], l, w, h, -(r + np.pi / 2)], axis=-1)


def frame_tables(prediction_infos, gt_infos, class_name, distance_thresh=100, fake_gt_infos=True):
    """The padded host tables of detection_metrics from the reference's frame dicts, by generate_waymo_type_results and
    mask_by_distance: ground-truth rows kept when their name is in class_name and num_points_in_gt > 0, difficulty 0 -> 1 (more than
    5 points) or 2, the fake-lidar conversion with fake_gt_infos, headings through limit_period(h, 0.5, 2 pi) and boxes kept where
    ||(x, y)|| < distance_thresh + 0.5, each on the concatenation of every frame's rows (so in its dtype), scores through a sigmoid
    when their maximum exceeds 1.  The inputs are not modified.  Returns a dict of numpy arrays pred, pred_cnt, gt_box, gt_type,
    gt_level, gt_cnt."""
    if len(prediction_infos) != len(gt_infos):
        raise ValueError('%d prediction frames vs %d ground-truth frames' % (len(prediction_infos), len(gt_infos)))
    NF = len(gt_infos)
    pf, pb, ps, pt, gf, gb, gt, gd = [], [], [], [], [], [], [], []
    for i, (pinfo, ginfo) in enumerate(zip(prediction_infos, gt_infos)):
        pb.append(pinfo['boxes_lidar'][:, :7])
        ps.append(pinfo['score'])
        pt += [WAYMO_CLASSES.index(x) for x in pinfo['name']]
        pf.append(np.full(len(pinfo['boxes_lidar']), i))
        names, npts = np.asarray(ginfo['name']), np.asarray(ginfo['num_points_in_gt'])
        diff = np.array(ginfo['difficulty'], copy=True)
        zero = diff == 0
        diff[(npts > 5) & zero] = 1
        diff[(npts <= 5) & zero] = 2
        keep = np.array([x in class_name for x in names], dtype=np.bool_) & (npts > 0)
        boxes = _fakelidar_to_lidar(ginfo['gt_boxes_lidar']) if fake_gt_infos else np.asarray(ginfo['gt_boxes_lidar'])
        gb.append(boxes[keep][:, :7])
        gt += [WAYMO_CLASSES.index(x) for x in names[keep]]
        gd.append(diff[keep])
        gf.append(np.full(int(keep.sum()), i))
    cat = lambda a, shape: np.concatenate(a, 0) if a else np.zeros(shape)
    pf, pb, ps, pt = cat(pf, (0,)).astype(np.int64), cat(pb, (0, 7)), cat(ps, (0,)).reshape(-1), np.array(pt, np.int64)
    gf, gb, gt, gd = cat(gf, (0,)).astype(np.int64), cat(gb, (0, 7)), np.array(gt, np.int64), cat(gd, (0,))
    pb[:, -1] = _limit_period(pb[:, -1], offset=0.5, period=np.pi * 2)
    gb[:, -1] = _limit_period(gb[:, -1], offset=0.5, period=np.pi * 2)
    pm = np.linalg.norm(pb[:, 0:2], axis=1) < distance_thresh + 0.5
    gm = np.linalg.norm(gb[:, 0:2], axis=1) < distance_thresh + 0.5
    pf, pb, ps, pt = pf[pm], pb[pm], ps[pm], pt[pm]
    gf, gb, gt, gd = gf[gm], gb[gm], gt[gm], gd[gm]
    if ps.size and ps.max() > 1:
        ps = 1 / (1 + np.exp(-ps))

    def pad(frame, cols):
        cnt = np.bincount(frame, minlength=NF).astype(np.int32)
        slot = np.arange(len(frame)) - (np.cumsum(cnt) - cnt)[frame]      # rows stay in frame order after the concatenation
        out = np.zeros((NF, max(int(cnt.max()) if NF else 0, 1), cols.shape[1]), np.float32)
        out[frame, slot] = cols
        return out, cnt
    pred, pred_cnt = pad(pf, np.concatenate([pb, ps[:, None], pt[:, None]], 1).astype(np.float32))
    g, gt_cnt = pad(gf, np.concatenate([gb, gt[:, None], gd[:, None]], 1).astype(np.float32))
    return {'pred': pred, 'pred_cnt': pred_cnt, 'gt_box': np.ascontiguousarray(g[..., :7]), 'gt_type': g[..., 7].astype(np.int32),
            'gt_level': g[..., 8].astype(np.int32), 'gt_cnt': gt_cnt}


class WaymoDetectionMetricsEstimator:
    """WaymoDetectionMetricsEstimator of waymo_eval_detection.py with the metric on the device.  After a call, ``records`` holds the
    records (16, 2, 101, 4) it was computed from."""
    WAYMO_CLASSES = WAYMO_CLASSES

    def __init__(self, device='cuda', max_pairs=1 << 14, frame_chunk=None):
        self.device, self.max_pairs, self.frame_chunk = device, max_pairs, frame_chunk
        self.records = None

    def waymo_evaluation(self, prediction_infos, gt_infos, class_name, config_type=['object'], distance_thresh=100,
                         fake_gt_infos=True):
        """prediction_infos: per frame {'boxes_lidar' (n, 7), 'score' (n), 'name' (n)} (io.load_result_pkl and
        OffboardResult.to_reference produce them); gt_infos: per frame the 'annos' of waymo_infos ('name', 'difficulty',
        'num_points_in_gt', 'gt_boxes_lidar'); config_type from 'object', 'range', '3d', 'bev'.  Returns the AP dict
        {key: [value]}, keys as the reference's (AP and APH only)."""
        breakdowns, box_type = _config(config_type)
        t = frame_tables(prediction_infos, gt_infos, class_name, distance_thresh, fake_gt_infos)
        d = {k: torch.from_numpy(np.ascontiguousarray(v)).to(self.device) for k, v in t.items()}
        self.records, ap = detection_metrics(d['pred'], d['pred_cnt'], d['gt_box'], d['gt_type'], d['gt_level'], d['gt_cnt'], box_type,
                                             breakdowns, self.max_pairs, self.frame_chunk)
        return ap


def _wrap_heading(h):
    period = torch.full_like(h, np.float32(np.pi * 2))        # a tensor divisor: torch divides a scalar by its reciprocal
    return h - torch.floor(h / period + 0.5) * np.float32(np.pi * 2)


def evaluate_offboard(results, gt, class_name=CLASS_NAMES, config_type=('object',), distance_thresh=1000, max_pairs=1 << 14,
                      frame_chunk=None, return_records=False):
    """AP / APH of offboard.refine_sequence's final boxes against ground truth, on the device: results, a list of OffboardResult
    (one per sequence of ``gt``, a track.GroundTruth of the same frames, in order).  The tables are prepared as frame_tables does,
    with torch elementwise ops in float32: predictions of every class (label 1..3 -> Waymo types 1, 2, 4), ground-truth rows of the
    classes in class_name with num_points > 0, difficulty 0 remapped by num_points, headings wrapped, rows beyond distance_thresh
    + 0.5 m dropped, scores through a sigmoid when their maximum exceeds 1 (selected on the device).  Ground-truth boxes are taken
    as they are (detzero_eval.py without --info_with_fakelidar).  Returns the AP dict (and the records with return_records)."""
    breakdowns, box_type = _config(config_type)
    for c in class_name:
        if c not in CLASS_NAMES:
            raise ValueError('class %r is not one of %r' % (c, CLASS_NAMES))
    S, F, G, _ = gt.box.shape
    if len(results) != S:
        raise ValueError('%d results for %d ground-truth sequences' % (len(results), S))
    dev = gt.box.device
    R = max([r.rows.shape[1] for r in results] + [1])
    pred = torch.zeros((S, F, R, 9), dtype=torch.float32, device=dev)
    pred_cnt = torch.zeros((S, F), dtype=torch.int32, device=dev)
    for s, r in enumerate(results):
        n = r.rows.shape[0]
        if n != len(gt.frame_ids[s]):
            raise ValueError('sequence %d: %d result frames against %d ground-truth frames' % (s, n, len(gt.frame_ids[s])))
        pred[s, :n, :r.rows.shape[1]] = r.rows
        pred_cnt[s, :n] = r.count.to(torch.int32)
    thr = np.float32(distance_thresh + 0.5)
    label_type = torch.tensor([0, 1, 2, 4], dtype=torch.float32, device=dev)
    row = torch.arange(R, device=dev)
    valid = row[None, None, :] < pred_cnt[..., None].long()
    x, y = pred[..., 0], pred[..., 1]
    keep = valid & (torch.sqrt(x * x + y * y) < thr)
    score = pred[..., 7]
    top = torch.where(keep, score, torch.full_like(score, -np.inf)).max()
    score = torch.where(top > 1, 1 / (1 + torch.exp(-score)), score)
    ptype = torch.where(keep, label_type[pred[..., 8].long().clamp(0, 3)], torch.zeros_like(score))
    pred = torch.cat([pred[..., :6], _wrap_heading(pred[..., 6:7]), score[..., None], ptype[..., None]], -1)
    cls_type = torch.tensor([0, 1, 2, 4], dtype=torch.int32, device=dev)
    sel = torch.zeros(4, dtype=torch.bool, device=dev)
    sel[[CLASS_NAMES.index(c) + 1 for c in class_name]] = True
    gvalid = torch.arange(G, device=dev)[None, None, :] < gt.counts[..., None].long()
    gx, gy = gt.box[..., 0], gt.box[..., 1]
    gkeep = gvalid & sel[gt.cls.long()] & (gt.num_points > 0) & (torch.sqrt(gx * gx + gy * gy) < thr)
    gtype = torch.where(gkeep, cls_type[gt.cls.long()], torch.zeros_like(gt.cls))
    level = torch.where(gt.difficulty == 0, torch.where(gt.num_points > 5, 1, 2), gt.difficulty).to(torch.int32)
    gbox = torch.cat([gt.box[..., :6], _wrap_heading(gt.box[..., 6:7])], -1)
    rec, ap = detection_metrics(pred.reshape(S * F, R, 9), pred_cnt.reshape(-1), gbox.reshape(S * F, G, 7), gtype.reshape(S * F, G),
                                level.reshape(S * F, G), gt.counts.reshape(-1), box_type, breakdowns, max_pairs, frame_chunk)
    return (ap, rec) if return_records else ap


# ------------------------------------------------------------------------------------------------------------------- tracking
#: WAYMO_CLASSES of the reference's tracking evaluator (waymo_eval_tracking.py): type 3 is 'Sign'
TRACKING_WAYMO_CLASSES = ['unknown', 'Vehicle', 'Pedestrian', 'Sign', 'Cyclist']
MOT_KEYS = ('MOTA', 'MOTP', 'MISS', 'MISMATCH', 'FP')


def _breakdowns(config_type):
    for c in config_type:
        if c not in ('object', 'range'):
            raise ValueError('unknown config type %r (supported: object, range)' % (c,))
    return tuple(b for b in ('object', 'range') if b in config_type)


def mot_dict(records, breakdowns=('object',)):
    """{'OBJECT_TYPE_TYPE_VEHICLE_LEVEL_1/MOTA': [v], ... /MOTP, /MISS, /MISMATCH, /FP, 'RANGE_TYPE_CYCLIST_[50, +inf)_LEVEL_2/FP':
    [v], ...} from the tracking records (16, 2, 101, 5), per shard and level at the cutoff with the largest MOTA (the lowest cutoff
    on a tie): MOTA = 1 - (misses + mismatches + FP) / num_gt, MOTP = cost / matches (0 without matches), MISS, MISMATCH, FP = each
    count / num_gt, num_gt = matches + misses; a shard with num_gt = 0 gets 0 everywhere.  SIGN keys are always present."""
    rec = np.asarray(records)
    shards = []
    if 'object' in breakdowns:
        shards += [(t, 'OBJECT_TYPE_TYPE_%s' % TYPE_NAMES[t]) for t in range(4)]
    if 'range' in breakdowns:
        shards += [(4 + 3 * t + r, 'RANGE_TYPE_%s_%s' % (TYPE_NAMES[t], RANGE_NAMES[r])) for t in range(4) for r in range(3)]
    out = {}
    for s, name in shards:
        for lvl in (0, 1):
            m, miss, fp, mm, cost = (rec[s, lvl, :, i].astype(np.float64) for i in range(5))
            n = m + miss
            if n[0] == 0:
                vals = [0.0] * 5
            else:
                mota = 1.0 - (miss + mm + fp) / n
                k = int(np.argmax(mota))
                vals = [float(mota[k]), float(cost[k] / _FIXED / m[k]) if m[k] else 0.0, float(miss[k] / n[k]), float(mm[k] / n[k]),
                        float(fp[k] / n[k])]
            for key, v in zip(MOT_KEYS, vals):
                out['%s_LEVEL_%d/%s' % (name, lvl + 1, key)] = [v]
    return out


def tracking_metrics(pred, pred_id, pred_cnt, gt_box, gt_obj, gt_type, gt_level, gt_cnt, num_frames=None, n_obj=None,
                     breakdowns=('object',), max_pairs=1 << 14):
    """Tracking records and MOTA / MOTP dict of S sequences on the device (csrc/track_eval.cu).  pred (S, F, R, 9) f32 CUDA [x, y, z,
    dx, dy, dz, heading, score, Waymo type], pred_id (S, F, R) int32 identity per sequence, pred_cnt (S, F) rows per frame; gt_box
    (S, F, G, 7) f32, gt_obj (S, F, G) per-sequence object index, gt_type (S, F, G) Waymo type, gt_level (S, F, G) 1 or 2, gt_cnt
    (S, F); num_frames (S) frames per sequence (default F), n_obj (S) objects per sequence (default 1 + the largest index).  Rows of a
    type outside 1..4 are ignored.  breakdowns from 'object', 'range'.  max_pairs: capacity of valid pairs of one type per frame.
    Raises ValueError when two rows of a frame share an id or an object index is out of range, RuntimeError past a capacity.
    Returns (records (16, 2, 101, 5) int64 numpy [shard][level][cutoff][matches, misses, FP, mismatches, cost in 2^-32 units],
    mot_dict); one device-to-host copy."""
    for b in breakdowns:
        if b not in ('object', 'range'):
            raise ValueError('unknown breakdown %r' % (b,))
    assert pred.is_cuda and pred.dtype == torch.float32 and pred.dim() == 4 and pred.shape[3] == 9, (pred.shape, pred.dtype)
    assert gt_box.is_cuda and gt_box.dtype == torch.float32 and gt_box.dim() == 4 and gt_box.shape[3] == 7, (gt_box.shape, gt_box.dtype)
    S, F, dev = pred.shape[0], pred.shape[1], pred.device
    if tuple(gt_box.shape[:2]) != (S, F):
        raise ValueError('predictions of %d sequences x %d frames against ground truth of %d x %d' % (S, F, *gt_box.shape[:2]))
    i32 = lambda t: torch.as_tensor(t).to(device=dev, dtype=torch.int32).contiguous()
    pred_id, pred_cnt, gt_obj, gt_type, gt_level, gt_cnt = (i32(t) for t in (pred_id, pred_cnt, gt_obj, gt_type, gt_level, gt_cnt))
    pred_cnt, gt_cnt = pred_cnt.reshape(S, F), gt_cnt.reshape(S, F)
    nf = torch.full((S,), F, dtype=torch.int32, device=dev) if num_frames is None else i32(num_frames).reshape(S)
    if n_obj is None:
        n_obj = (gt_obj.reshape(S, -1).amax(1) + 1).clamp(min=0) if gt_obj.numel() else torch.zeros(S, dtype=torch.int32, device=dev)
    n_obj = i32(n_obj).reshape(S)
    if pred.shape[2] == 0:
        pred, pred_id, pred_cnt = (torch.zeros((S, F, 1, 9), dtype=torch.float32, device=dev), torch.zeros((S, F, 1), **_I32(dev)),
                                   torch.zeros_like(pred_cnt))
    if gt_box.shape[2] == 0:
        gt_box, gt_cnt = torch.zeros((S, F, 1, 7), dtype=torch.float32, device=dev), torch.zeros_like(gt_cnt)
        gt_obj = gt_type = gt_level = torch.zeros((S, F, 1), **_I32(dev))
    pred, gt_box = pred.contiguous(), gt_box.contiguous()
    R, G = pred.shape[2], gt_box.shape[2]
    for name, t in (('pred_id', pred_id), ('gt_obj', gt_obj), ('gt_type', gt_type), ('gt_level', gt_level)):
        if tuple(t.shape) != (S, F, R if name == 'pred_id' else G):
            raise ValueError('%s must be (S, F, %s)' % (name, 'R' if name == 'pred_id' else 'G'))
    O = max(int(n_obj.max()) if S else 0, 1)
    records = torch.zeros((16, 2, NUM_CUTOFFS, 5), dtype=torch.int64, device=dev)
    flags = torch.zeros((1,), dtype=torch.int32, device=dev)
    mask = sum(1 << i for i, b in enumerate(('object', 'range')) if b in breakdowns)
    if S and mask:
        ws = ops.workspace(lib().dz_track_eval_ws_bytes(S, R, G, O, int(max_pairs)), dev, 'track_eval')
        check(lib().dz_track_eval(ops._p(pred), ops._p(pred_id), ops._p(pred_cnt), ops._p(gt_box), ops._p(gt_obj), ops._p(gt_type),
                                  ops._p(gt_level), ops._p(gt_cnt), ops._p(nf), ops._p(n_obj), S, F, R, G, O, mask, int(max_pairs),
                                  ops._p(records), ops._p(flags), ops._p(ws), ws.numel(), ops._stream()), 'track_eval')
        ops._count(1)
    out = torch.cat([records.reshape(-1), flags.long()]).cpu().numpy()
    rec, fl = out[:-1].reshape(16, 2, NUM_CUTOFFS, 5), int(out[-1])
    if fl & 12:
        what = [n for b, n in ((4, 'two rows of one frame share an id'), (8, 'a ground-truth object index is outside [0, n_obj)'))
                if fl & b]
        raise ValueError('track_eval: %s' % '; '.join(what))
    if fl & 3:
        what = [n for b, n in ((1, 'valid pairs per frame (max_pairs=%d)' % max_pairs), (2, 'the assignment scratch')) if fl & b]
        raise RuntimeError('track_eval: a frame exceeded the capacity of %s' % ', '.join(what))
    return rec, mot_dict(rec, breakdowns)


def _I32(dev):
    return dict(dtype=torch.int32, device=dev)


def tracking_tables(prediction_infos, gt_infos, class_name, fake_gt_infos=True):
    """The padded host tables of tracking_metrics from the reference's frame dicts, by generate_waymo_type_results:
    prediction_infos per frame {'sequence_name', 'obj_ids', 'boxes_lidar', 'score', 'name'}, gt_infos per frame {'sequence_name',
    'annos': {'name', 'obj_ids', 'difficulty', 'num_points_in_gt', 'gt_boxes_lidar'}}, frame i of both lists the same frame.
    Ground-truth rows kept when their name is in class_name and num_points_in_gt > 0, difficulty 0 -> 1 (more than 5 points) or 2,
    the fake-lidar conversion with fake_gt_infos, headings through limit_period(h, 0.5, 2 pi) on the concatenation of every frame's
    rows, scores through a sigmoid when their maximum exceeds 1.  Names map through TRACKING_WAYMO_CLASSES (an unknown name raises
    ValueError, as list.index does).  Prediction ids are sequence_name + '-' + str(obj_id), numbered per sequence (of the ground
    truth's sequence_name) in order of first appearance, as are ground-truth obj_ids.  A sequence's frames keep their list order,
    also when sequences interleave.  A prediction frame whose obj_ids and boxes_lidar differ in length raises ValueError (frames
    with dropped detections, which have no identity).  The inputs are not modified.  Returns a dict of numpy arrays pred, pred_id,
    pred_cnt, gt_box, gt_obj, gt_type, gt_level, gt_cnt, num_frames, n_obj, and 'sequences' (names in order of first frame)."""
    if len(prediction_infos) != len(gt_infos):
        raise ValueError('%d prediction frames vs %d ground-truth frames' % (len(prediction_infos), len(gt_infos)))
    NF = len(gt_infos)
    seq_names = list(dict.fromkeys(info['sequence_name'] for info in gt_infos))
    sidx = {n: i for i, n in enumerate(seq_names)}
    S = len(seq_names)
    fseq = np.array([sidx[info['sequence_name']] for info in gt_infos], np.int64)
    nfr = np.bincount(fseq, minlength=S).astype(np.int32)
    fpos = np.zeros(NF, np.int64)
    for s in range(S):
        fpos[fseq == s] = np.arange(nfr[s])
    pf, pb, ps, pt, pk, gf, gb, gt, gd, gk = [], [], [], [], [], [], [], [], [], []
    for i, (pinfo, info) in enumerate(zip(prediction_infos, gt_infos)):
        n = len(pinfo['boxes_lidar'])
        ids = pinfo['obj_ids'] if n or 'obj_ids' in pinfo else []
        if len(ids) != n:
            raise ValueError('prediction frame %d has %d obj_ids for %d boxes_lidar (dropped detections have no identity)'
                             % (i, len(ids), n))
        pb.append(np.asarray(pinfo['boxes_lidar'])[:, :7].reshape(-1, 7))
        ps.append(np.asarray(pinfo['score']).reshape(-1))
        pt += [TRACKING_WAYMO_CLASSES.index(x) for x in pinfo['name']]
        pk += [(fseq[i], pinfo['sequence_name'] + '-' + str(x)) for x in ids]
        pf.append(np.full(n, i))
        a = info['annos']
        names, npts = np.asarray(a['name']), np.asarray(a['num_points_in_gt'])
        diff = np.array(a['difficulty'], copy=True)
        zero = diff == 0
        diff[(npts > 5) & zero] = 1
        diff[(npts <= 5) & zero] = 2
        keep = np.array([x in class_name for x in names], dtype=np.bool_) & (npts > 0)
        boxes = _fakelidar_to_lidar(a['gt_boxes_lidar']) if fake_gt_infos else np.asarray(a['gt_boxes_lidar'])
        gb.append(boxes[keep][:, :7])
        gt += [TRACKING_WAYMO_CLASSES.index(x) for x in names[keep]]
        gd.append(diff[keep])
        gk += [(fseq[i], x) for x in np.asarray(a['obj_ids'])[keep]]
        gf.append(np.full(int(keep.sum()), i))
    cat = lambda a, shape: np.concatenate(a, 0) if a else np.zeros(shape)
    pf, pb, ps, pt = cat(pf, (0,)).astype(np.int64), cat(pb, (0, 7)), cat(ps, (0,)).reshape(-1), np.array(pt, np.int64)
    gf, gb, gt, gd = cat(gf, (0,)).astype(np.int64), cat(gb, (0, 7)), np.array(gt, np.int64), cat(gd, (0,))
    pb[:, -1] = _limit_period(pb[:, -1], offset=0.5, period=np.pi * 2)
    gb[:, -1] = _limit_period(gb[:, -1], offset=0.5, period=np.pi * 2)
    if ps.size and ps.max() > 1:
        ps = 1 / (1 + np.exp(-ps))
    pidx, gidx = [{} for _ in range(S)], [{} for _ in range(S)]
    pid = np.array([pidx[s].setdefault(k, len(pidx[s])) for s, k in pk], np.int64)
    gobj = np.array([gidx[s].setdefault(k, len(gidx[s])) for s, k in gk], np.int64)
    F = max(int(nfr.max()) if S else 0, 1)

    def pad(frame, cols):
        cnt = np.bincount(frame, minlength=NF).astype(np.int32)
        slot = np.arange(len(frame)) - (np.cumsum(cnt) - cnt)[frame]
        out = np.zeros((S, F, max(int(cnt.max()) if NF else 0, 1), cols.shape[1]), np.float64)
        out[fseq[frame], fpos[frame], slot] = cols
        c = np.zeros((S, F), np.int32)
        c[fseq, fpos] = cnt
        return out, c
    p, pred_cnt = pad(pf, np.concatenate([pb.astype(np.float32).astype(np.float64), ps.astype(np.float32)[:, None], pt[:, None],
                                          pid[:, None]], 1))
    g, gt_cnt = pad(gf, np.concatenate([gb.astype(np.float32).astype(np.float64), gt[:, None], gd[:, None], gobj[:, None]], 1))
    return {'pred': np.ascontiguousarray(p[..., :9].astype(np.float32)), 'pred_id': p[..., 9].astype(np.int32), 'pred_cnt': pred_cnt,
            'gt_box': np.ascontiguousarray(g[..., :7].astype(np.float32)), 'gt_type': g[..., 7].astype(np.int32),
            'gt_level': g[..., 8].astype(np.int32), 'gt_obj': g[..., 9].astype(np.int32), 'gt_cnt': gt_cnt, 'num_frames': nfr,
            'n_obj': np.array([len(d) for d in gidx], np.int32), 'sequences': seq_names}


class WaymoTrackingMetricsEstimator:
    """WaymoTrackingMetricsEstimator of waymo_eval_tracking.py with the metric on the device (csrc/track_eval.cu).  After a call,
    ``records`` holds the records (16, 2, 101, 5) it was computed from."""
    WAYMO_CLASSES = TRACKING_WAYMO_CLASSES

    def __init__(self, device='cuda', max_pairs=1 << 14):
        self.device, self.max_pairs = device, max_pairs
        self.records = None

    def waymo_evaluation(self, prediction_infos, gt_infos, class_name, config_type=['object'], distance_thresh=100,
                         fake_gt_infos=True):
        """prediction_infos / gt_infos as tracking_tables takes them (detzero_eval.py --tracking passes the full ground-truth infos);
        config_type from 'object', 'range'.  distance_thresh is accepted and ignored, as the reference's mask_by_distance keeps every
        box.  Returns the metric dict {key: [value]}, keys as the reference's (MOTA, MOTP, MISS, MISMATCH, FP)."""
        breakdowns = _breakdowns(config_type)
        t = tracking_tables(prediction_infos, gt_infos, class_name, fake_gt_infos)
        d = {k: torch.from_numpy(np.ascontiguousarray(v)).to(self.device) for k, v in t.items() if k != 'sequences'}
        self.records, out = tracking_metrics(d['pred'], d['pred_id'], d['pred_cnt'], d['gt_box'], d['gt_obj'], d['gt_type'],
                                             d['gt_level'], d['gt_cnt'], d['num_frames'], d['n_obj'], breakdowns, self.max_pairs)
        return out


def _gt_tracking_tables(gt, class_name):
    """ground-truth tables of tracking_metrics from a track.GroundTruth: rows of the classes in class_name with num_points > 0 (others
    get type 0), difficulty 0 remapped by num_points, headings wrapped; boxes as they are (no fake-lidar conversion)"""
    for c in class_name:
        if c not in CLASS_NAMES:
            raise ValueError('class %r is not one of %r' % (c, CLASS_NAMES))
    dev = gt.box.device
    G = gt.box.shape[2]
    cls_type = torch.tensor([0, 1, 2, 4], dtype=torch.int32, device=dev)
    sel = torch.zeros(4, dtype=torch.bool, device=dev)
    sel[[CLASS_NAMES.index(c) + 1 for c in class_name]] = True
    gvalid = torch.arange(G, device=dev)[None, None, :] < gt.counts[..., None].long()
    gkeep = gvalid & sel[gt.cls.long()] & (gt.num_points > 0)
    gtype = torch.where(gkeep, cls_type[gt.cls.long()], torch.zeros_like(gt.cls))
    level = torch.where(gt.difficulty == 0, torch.where(gt.num_points > 5, 1, 2), gt.difficulty).to(torch.int32)
    gbox = torch.cat([gt.box[..., :6], _wrap_heading(gt.box[..., 6:7])], -1)
    return gbox, gt.obj, gtype, level


def _pred_finish(pred, pred_cnt, label_type):
    """scores through a sigmoid when the maximum over the rows exceeds 1 (selected on the device), headings wrapped, the label
    column replaced by its Waymo type"""
    R = pred.shape[2]
    valid = torch.arange(R, device=pred.device)[None, None, :] < pred_cnt[..., None].long()
    score = pred[..., 7]
    top = torch.where(valid, score, torch.full_like(score, -np.inf)).max() if pred.numel() else score.new_tensor(0.)
    score = torch.where(top > 1, 1 / (1 + torch.exp(-score)), score)
    ptype = torch.where(valid, label_type, torch.zeros_like(score))
    return torch.cat([pred[..., :6], _wrap_heading(pred[..., 6:7]), score[..., None], ptype[..., None]], -1)


def track_tables(track_result, gt, class_name=CLASS_NAMES):
    """The device tables of tracking_metrics (a dict of its argument names) for a track.TrackResult against a track.GroundTruth of
    the same sequences and frames.  Every entry of every track is a prediction at its frame, as daemon/combine_output.py
    convert_frame_format places it: its world box back in the frame's lidar frame (the conversion of csrc/track_gt.cu), the entry's
    score, the track's class (Waymo types 1, 2, 4) and the track id as its identity.  Ground-truth rows of the classes in class_name
    with num_points > 0, difficulty 0 remapped by num_points, boxes as they are (no fake-lidar conversion); headings wrapped and
    scores through a sigmoid when their maximum exceeds 1, as tracking_tables does.  Built with torch ops on the device, no host loop
    over entries."""
    gbox, gobj, gtype, level = _gt_tracking_tables(gt, class_name)
    S, F = gt.box.shape[:2]
    trk = track_result.trk
    if trk.shape[0] != S or track_result.poses.shape[1] != F:
        raise ValueError('tracks of %d sequences / %d frames against ground truth of %d / %d' % (trk.shape[0],
                                                                                              track_result.poses.shape[1], S, F))
    dev = gt.box.device
    E = track_result.ent_box.shape[1]
    ent_frame = track_result.ent_frame.to(torch.int32).contiguous()
    nf = track_result.num_frames.to(device=dev, dtype=torch.int32).contiguous()
    lidar = torch.empty((S, E, 7), dtype=torch.float32, device=dev)
    check(lib().dz_track_entry_lidar(ops._p(track_result.ent_box.contiguous()), ops._p(ent_frame),
                                     ops._p(track_result.poses.to(torch.float64).contiguous()), ops._p(nf), S, E, F, ops._p(lidar),
                                     ops._stream()), 'track_entry_lidar')
    ops._count(1)
    nt = torch.as_tensor(np.asarray(track_result.n_tracks, np.int64), device=dev)
    T = trk.shape[1]
    tvalid = torch.arange(T, device=dev)[None, :] < nt[:, None]
    off = torch.where(tvalid, trk[..., 5].long(), torch.full_like(trk[..., 5].long(), 1 << 40))
    n_ent = torch.where(tvalid, trk[..., 5].long() + trk[..., 3].long(), torch.zeros_like(off)).amax(1) if T else nt
    e = torch.arange(E, device=dev)
    k = (torch.searchsorted(off.contiguous(), e[None, :].expand(S, E).contiguous(), right=True) - 1).clamp(0, max(T - 1, 0))
    ef = ent_frame.long()
    valid = (e[None, :] < n_ent[:, None]) & (ef >= 0) & (ef < nf.long()[:, None])
    cell = (torch.arange(S, device=dev)[:, None] * F + ef)[valid]
    order = torch.sort(cell, stable=True).indices
    cell = cell[order]
    cnt = torch.bincount(cell, minlength=S * F)
    R = max(int(cnt.max()) if cell.numel() else 0, 1)
    slot = torch.arange(cell.numel(), device=dev) - (torch.cumsum(cnt, 0) - cnt)[cell]
    label_type = torch.tensor([0, 1, 2, 4], dtype=torch.float32, device=dev)
    cls = torch.gather(trk[..., 1].long(), 1, k)[valid][order]
    rows = torch.cat([lidar[valid][order], track_result.ent_score[valid][order].float()[:, None], cls.float()[:, None]], 1)
    pred = torch.zeros((S * F, R, 9), dtype=torch.float32, device=dev)
    pred[cell, slot] = rows
    pred_id = torch.zeros((S * F, R), dtype=torch.int32, device=dev)
    pred_id[cell, slot] = torch.gather(trk[..., 0], 1, k)[valid][order]
    pred_cnt = cnt.reshape(S, F).to(torch.int32)
    pred = pred.reshape(S, F, R, 9)
    pred = _pred_finish(pred, pred_cnt, label_type[pred[..., 8].long().clamp(0, 3)])
    return {'pred': pred, 'pred_id': pred_id.reshape(S, F, R), 'pred_cnt': pred_cnt, 'gt_box': gbox, 'gt_obj': gobj, 'gt_type': gtype,
            'gt_level': level, 'gt_cnt': gt.counts, 'num_frames': gt.num_frames, 'n_obj': gt.n_obj}


def evaluate_tracks(track_result, gt, class_name=CLASS_NAMES, config_type=('object',), max_pairs=1 << 14, return_records=False):
    """MOTA / MOTP of the raw tracker output (track.track_sequences) against ground truth, on the device: track_result a
    track.TrackResult and gt a track.GroundTruth of the same sequences and frames, tables by track_tables.  Returns the metric dict
    (and the records with return_records)."""
    breakdowns = _breakdowns(config_type)
    rec, out = tracking_metrics(**track_tables(track_result, gt, class_name), breakdowns=breakdowns, max_pairs=max_pairs)
    return (out, rec) if return_records else out


def evaluate_offboard_tracking(results, gt, class_name=CLASS_NAMES, config_type=('object',), max_pairs=1 << 14, return_records=False):
    """MOTA / MOTP of offboard.refine_sequence's final boxes against ground truth, on the device: results a list of OffboardResult
    (one per sequence of ``gt``, a track.GroundTruth of the same frames, in order).  The track rows (obj_id >= 0) are the
    predictions, with the track id as their identity; dropped detections (obj_id -1) have no identity and are left out.
    Labels 1..3 map to Waymo types 1, 2, 4; ground truth as evaluate_tracks takes it.  Returns the metric dict (and the records
    with return_records)."""
    breakdowns = _breakdowns(config_type)
    gbox, gobj, gtype, level = _gt_tracking_tables(gt, class_name)
    S, F = gt.box.shape[:2]
    if len(results) != S:
        raise ValueError('%d results for %d ground-truth sequences' % (len(results), S))
    dev = gt.box.device
    R = max([r.rows.shape[1] for r in results] + [1])
    pred = torch.zeros((S, F, R, 9), dtype=torch.float32, device=dev)
    pred_id = torch.zeros((S, F, R), dtype=torch.int32, device=dev)
    pred_cnt = torch.zeros((S, F), dtype=torch.int32, device=dev)
    for s, r in enumerate(results):
        n = r.rows.shape[0]
        if n != len(gt.frame_ids[s]):
            raise ValueError('sequence %d: %d result frames against %d ground-truth frames' % (s, n, len(gt.frame_ids[s])))
        w = r.rows.shape[1]
        live = torch.arange(w, device=dev)[None, :] < r.count.to(dev).long()[:, None]
        pred[s, :n, :w] = r.rows
        pred_id[s, :n, :w] = r.obj_id.to(torch.int32)
        pred_cnt[s, :n] = ((r.obj_id >= 0) & live).sum(1).to(torch.int32)     # the track rows come first
    label_type = torch.tensor([0, 1, 2, 4], dtype=torch.float32, device=dev)
    pred = _pred_finish(pred, pred_cnt, label_type[pred[..., 8].long().clamp(0, 3)])
    rec, out = tracking_metrics(pred, pred_id, pred_cnt, gbox, gobj, gtype, level, gt.counts, gt.num_frames, gt.n_obj, breakdowns,
                                max_pairs)
    return (out, rec) if return_records else out

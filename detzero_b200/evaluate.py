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
distant recall points."""
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

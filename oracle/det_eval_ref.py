"""Plain numpy restatement of the detection AP / APH metric of csrc/det_eval.cu and detzero_b200/evaluate.py (Waymo AP and APH per
object type, difficulty level and range, as DetZero's evaluator reports them), written for clarity: loops over frame x type x
cutoff, scipy's linear_sum_assignment on the valid-pair IoU matrix, float64 everywhere except where the definition says float32.

``waymo_evaluation`` restates the host preparation of WaymoDetectionMetricsEstimator.waymo_evaluation
(detection/detzero_det/datasets/waymo/waymo_eval_detection.py: generate_waymo_type_results, mask_by_distance) and returns
(ap dict, records, Margin); ``records`` takes already prepared frames.  The Margin holds the smallest |IoU - threshold|,
|score - cutoff| and |range - boundary| over the decisions taken, so a test can tell when a comparison with the device is not
decided by rounding."""
import numpy as np
from scipy.optimize import linear_sum_assignment

from . import boxes_iou3d, boxes_iou_bev
from .track_ref import Margin

WAYMO_CLASSES = ['unknown', 'Vehicle', 'Pedestrian', 'Truck', 'Cyclist']
TYPE_NAMES = ['VEHICLE', 'PEDESTRIAN', 'SIGN', 'CYCLIST']
RANGE_NAMES = ['[0, 30)', '[30, 50)', '[50, +inf)']
IOU_THRESH = {1: np.float32(0.7), 2: np.float32(0.5), 3: np.float32(0.5), 4: np.float32(0.5)}
CUTOFFS = np.array([np.float32(k * 0.01) for k in range(100)] + [np.float32(1.0)], np.float32)
FIXED = 2.0 ** 32


def range_of(box):
    x, y = np.float32(box[0]), np.float32(box[1])
    r = np.sqrt(x * x + y * y)
    return 0 if r < np.float32(30) else (1 if r < np.float32(50) else 2)


def heading_accuracy_fixed(h_pred, h_gt):
    d = np.fmod(float(np.float32(h_pred)) - float(np.float32(h_gt)), 2 * np.pi)
    if d < 0:
        d += 2 * np.pi
    acc = 1.0 - min(d, 2 * np.pi - d) / np.pi
    return int(np.rint(acc * FIXED))


def _match(iou, rows, cols, thr):
    """maximum-IoU-sum matching of ground truth ``rows`` and predictions ``cols`` over the pairs with IoU >= thr -> {row: col}"""
    if not len(rows) or not len(cols):
        return {}
    w = iou[np.ix_(rows, cols)].astype(np.float64)
    w = np.where(w >= thr, w, 0.0)
    r, c = linear_sum_assignment(w, maximize=True)
    return {rows[i]: cols[j] for i, j in zip(r, c) if w[i, j] > 0}


def records(frames, box_type='3d', breakdowns=('object',), margin=None):
    """frames: a list of (pred (n, 9) [box7, score, Waymo type], gt_box (m, 7), gt_type (m), gt_level (m)) -> records
    (16, 2, 101, 4) int64 [shard][level][cutoff][TP, FP, FN, TPH], and the Margin"""
    margin = Margin() if margin is None else margin
    rec = np.zeros((16, 2, 101, 4), np.int64)
    for pred, gbox, gtype, glevel in frames:
        pred = np.asarray(pred, np.float32).reshape(-1, 9)
        gbox = np.asarray(gbox, np.float32).reshape(-1, 7)
        gtype, glevel = np.asarray(gtype).reshape(-1), np.asarray(glevel).reshape(-1)
        ptype = pred[:, 8].astype(np.int64)
        prange = [range_of(b) for b in pred]
        grange = [range_of(b) for b in gbox]
        for b in list(pred) + list(gbox):
            x, y = np.float32(b[0]), np.float32(b[1])
            r = float(np.sqrt(x * x + y * y))
            margin.add([r, r], [30.0, 50.0], 'range')
        for s in pred[:, 7]:
            margin.add(CUTOFFS.astype(np.float64), float(s), 'score')
        for t in (1, 2, 3, 4):
            gi = [g for g in range(len(gbox)) if gtype[g] == t]
            pi = [p for p in range(len(pred)) if ptype[p] == t]
            iou = np.zeros((len(gbox), len(pred)), np.float32)
            if gi and pi:
                f = boxes_iou3d if box_type == '3d' else boxes_iou_bev
                sub = f(gbox[gi], pred[pi][:, :7])
                iou[np.ix_(gi, pi)] = sub
                margin.add(sub[sub > 0], float(IOU_THRESH[t]), 'iou')
            for k in range(101):
                active = [p for p in pi if pred[p, 7] >= CUTOFFS[k]]
                shards = []
                if 'object' in breakdowns:
                    shards.append((t - 1, [_match(iou, gi, active, IOU_THRESH[t])], gi, active))
                if 'range' in breakdowns:
                    ms = [_match(iou, [g for g in gi if grange[g] == r], active, IOU_THRESH[t]) for r in range(3)]
                    for r in range(3):
                        shards.append((4 + 3 * (t - 1) + r, [ms[r]], [g for g in gi if grange[g] == r],
                                       [p for p in active if prange[p] == r]))
                        shards[-1][1].extend(ms)          # FP: a prediction matched in none of the type's range matchings
                for shard, ms, gts, preds in shards:
                    m = ms[0]
                    matched_preds = set(p for mm in ms[1:] or ms for p in mm.values())
                    fp = sum(1 for p in preds if p not in matched_preds)
                    for lvl in (1, 2):
                        counts = [g for g in gts if (2 if glevel[g] == 2 else 1) <= lvl]
                        tp = [g for g in counts if g in m]
                        tph = sum(heading_accuracy_fixed(pred[m[g], 6], gbox[g, 6]) for g in tp)
                        rec[shard, lvl - 1, k] += [len(tp), fp, len(counts) - len(tp), tph]
    return rec, margin


def average_precision(tp, fp, fn, tph=None):
    """area under the precision envelope of the 101 (recall, precision) points, recall-sorted, from recall 0; with tph, the heading
    weighted TP replaces TP in the numerators"""
    num = tp if tph is None else tph
    pts = []
    for k in range(len(tp)):
        p = num[k] / (tp[k] + fp[k]) if tp[k] + fp[k] > 0 else 0.0
        r = num[k] / (tp[k] + fn[k]) if tp[k] + fn[k] > 0 else 0.0
        pts.append((r, p))
    order = sorted(range(len(pts)), key=lambda i: pts[i][0])
    ap, prev = 0.0, 0.0
    for i in order:
        r = pts[i][0]
        env = max(p2 for r2, p2 in pts if r2 >= r)
        ap += (r - prev) * env
        prev = r
    return ap


def ap_dict(rec, breakdowns=('object',)):
    """{'OBJECT_TYPE_TYPE_VEHICLE_LEVEL_1/AP': [ap], ..., 'RANGE_TYPE_VEHICLE_[0, 30)_LEVEL_1/APH': [aph], ...}"""
    out = {}
    shards = []
    if 'object' in breakdowns:
        shards += [(t, 'OBJECT_TYPE_TYPE_%s' % TYPE_NAMES[t]) for t in range(4)]
    if 'range' in breakdowns:
        shards += [(4 + 3 * t + r, 'RANGE_TYPE_%s_%s' % (TYPE_NAMES[t], RANGE_NAMES[r])) for t in range(4) for r in range(3)]
    for s, name in shards:
        for lvl in (0, 1):
            tp, fp, fn, tph = (rec[s, lvl, :, i].astype(np.float64) for i in range(4))
            if tp[0] + fn[0] == 0:
                ap = aph = 0.0
            else:
                ap, aph = average_precision(tp, fp, fn), average_precision(tp, fp, fn, tph / FIXED)
            out['%s_LEVEL_%d/AP' % (name, lvl + 1)] = [ap]
            out['%s_LEVEL_%d/APH' % (name, lvl + 1)] = [aph]
    return out


def limit_period(val, offset=0.5, period=np.pi):
    return val - np.floor(val / period + offset) * period


def fakelidar_to_lidar(b):
    b = np.array(b)
    w, l, h, r = b[:, 3:4], b[:, 4:5], b[:, 5:6], b[:, 6:7]
    b[:, 2] += h[:, 0] / 2
    return np.concatenate([b[:, 0:3], l, w, h, -(r + np.pi / 2)], axis=-1)


def prepare(prediction_infos, gt_infos, class_name, config_type=('object',), distance_thresh=100, fake_gt_infos=True):
    """the frames ``records`` takes, from the reference's frame dicts (inputs are not modified)"""
    for c in config_type:
        if c not in ('object', 'range', '3d', 'bev'):
            raise ValueError('unknown config type %r' % (c,))
    assert len(prediction_infos) == len(gt_infos)
    if not len(gt_infos):
        return []
    # every frame's rows are concatenated first, as the reference does: the dtype of the concatenation (float64 as soon as one
    # frame is, e.g. detzero_eval.py's empty entries) is the dtype of the heading wrap, the distance and the sigmoid
    pf, pb, ps, pt = [], [], [], []
    gf, gb, gt, gd = [], [], [], []
    for i, (pinfo, ginfo) in enumerate(zip(prediction_infos, gt_infos)):
        n = len(pinfo['boxes_lidar'])
        pb.append(pinfo['boxes_lidar'][:, :7])
        ps.append(pinfo['score'])
        pt += [WAYMO_CLASSES.index(x) for x in pinfo['name']]
        pf.append(np.full(n, i))
        names = np.asarray(ginfo['name'])
        npts = np.asarray(ginfo['num_points_in_gt'])
        diff = np.array(ginfo['difficulty'], copy=True)
        zero = diff == 0
        diff[zero & (npts > 5)] = 1
        diff[zero & (npts <= 5)] = 2
        keep = np.array([x in class_name for x in names], bool) & (npts > 0)
        boxes = np.array(ginfo['gt_boxes_lidar'])
        if fake_gt_infos:
            boxes = fakelidar_to_lidar(boxes)
        gb.append(boxes[keep][:, :7])
        gt += [WAYMO_CLASSES.index(x) for x in names[keep]]
        gd.append(diff[keep])
        gf.append(np.full(int(keep.sum()), i))
    pf, pb, ps, pt = np.concatenate(pf), np.concatenate(pb, 0), np.concatenate(ps).reshape(-1), np.array(pt, np.int64)
    gf, gb, gt, gd = np.concatenate(gf), np.concatenate(gb, 0), np.array(gt, np.int64), np.concatenate(gd)
    pb[:, -1] = limit_period(pb[:, -1], offset=0.5, period=np.pi * 2)
    gb[:, -1] = limit_period(gb[:, -1], offset=0.5, period=np.pi * 2)
    pm = np.linalg.norm(pb[:, 0:2], axis=1) < distance_thresh + 0.5
    gm = np.linalg.norm(gb[:, 0:2], axis=1) < distance_thresh + 0.5
    pf, pb, ps, pt = pf[pm], pb[pm], ps[pm], pt[pm]
    gf, gb, gt, gd = gf[gm], gb[gm], gt[gm], gd[gm]
    if ps.size and ps.max() > 1:
        ps = 1 / (1 + np.exp(-ps))
    frames = []
    for i in range(len(gt_infos)):
        p, g = pf == i, gf == i
        pred = np.zeros((int(p.sum()), 9), np.float32)
        pred[:, :7], pred[:, 7], pred[:, 8] = pb[p], ps[p], pt[p]
        frames.append((pred, gb[g].astype(np.float32), gt[g], gd[g]))
    return frames


def waymo_evaluation(prediction_infos, gt_infos, class_name, config_type=('object',), distance_thresh=100, fake_gt_infos=True):
    frames = prepare(prediction_infos, gt_infos, class_name, config_type, distance_thresh, fake_gt_infos)
    breakdowns = tuple(c for c in ('object', 'range') if c in config_type)
    rec, margin = records(frames, 'bev' if 'bev' in config_type and '3d' not in config_type else '3d', breakdowns)
    return ap_dict(rec, breakdowns), rec, margin

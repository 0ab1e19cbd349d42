"""Plain numpy restatement of the tracking MOTA / MOTP metric of csrc/track_eval.cu and detzero_b200/evaluate.py (Waymo MOTA, MOTP,
MISS, MISMATCH and FP per object type, difficulty level and range, as DetZero's evaluator reports them in tracking mode), written
for clarity: loops over sequence x type x cutoff x frame, scipy's linear_sum_assignment on the valid-pair IoU matrix.

The metric is CLEAR-MOT.  Matching runs per (sequence, Waymo type, cutoff) over the sequence's frames in order; per frame a pair
matched in the previous frame is kept while both are present, the prediction is active (score >= cutoff) and the pair is valid
(iou3d >= 0.7 vehicle, 0.5 otherwise); the rest is matched by the maximum IoU sum over valid pairs; a match is a mismatch when
its object was matched before (in any earlier frame) to another id.  At LEVEL_L a row counts when its level <= L: a match of a
counting row adds a match, 1 - IoU (float64, rounded to 2^-32 units) to the cost and possibly a mismatch; an unmatched counting
row is a miss; an unmatched active prediction an FP.  RANGE shards split the counts by the range of the ground-truth box (the
prediction's for an FP).

``waymo_evaluation`` restates the host preparation of WaymoTrackingMetricsEstimator.waymo_evaluation
(evaluator/waymo_eval_tracking.py: generate_waymo_type_results) and returns (metric dict, records, Margin); ``records`` takes
already prepared sequences.  The Margin holds the smallest |IoU - threshold|, |score - cutoff| and |range - boundary| over the
decisions taken."""
import numpy as np
from scipy.optimize import linear_sum_assignment

from . import boxes_iou3d
from .det_eval_ref import CUTOFFS, FIXED, IOU_THRESH, RANGE_NAMES, TYPE_NAMES, fakelidar_to_lidar, limit_period, range_of
from .track_ref import Margin

#: WAYMO_CLASSES of waymo_eval_tracking.py (type 3 is 'Sign')
WAYMO_CLASSES = ['unknown', 'Vehicle', 'Pedestrian', 'Sign', 'Cyclist']
FIELDS = ('matches', 'misses', 'fp', 'mismatches', 'cost')


def _check_unique(ids, what):
    ids = list(ids)
    if len(set(ids)) != len(ids):
        raise ValueError('two rows of one frame share a %s' % what)


def records(sequences, margin=None):
    """sequences: a list of sequences, each a list of frames (pred (n, 9) [box7, score, Waymo type], pred_id (n), gt_box (m, 7),
    gt_obj (m), gt_type (m), gt_level (m)) in order -> records (16, 2, 101, 5) int64 [shard][level][cutoff][matches, misses, FP,
    mismatches, cost], and the Margin"""
    margin = Margin() if margin is None else margin
    rec = np.zeros((16, 2, 101, 5), np.int64)
    for frames in sequences:
        pre = []
        for pred, pid, gbox, gobj, gtype, glevel in frames:
            pred = np.asarray(pred, np.float32).reshape(-1, 9)
            gbox = np.asarray(gbox, np.float32).reshape(-1, 7)
            gtype, glevel, gobj, pid = (np.asarray(a).reshape(-1) for a in (gtype, glevel, gobj, pid))
            ptype = pred[:, 8].astype(np.int64)
            pv, gv = (ptype >= 1) & (ptype <= 4), (gtype >= 1) & (gtype <= 4)
            _check_unique(pid[pv], 'prediction id')
            _check_unique(gobj[gv], 'ground-truth object')
            for b in list(pred) + list(gbox):
                x, y = np.float32(b[0]), np.float32(b[1])
                r = float(np.sqrt(x * x + y * y))
                margin.add([r, r], [30.0, 50.0], 'range')
            for s in pred[:, 7]:
                margin.add(CUTOFFS.astype(np.float64), float(s), 'score')
            per_type = {}
            for t in (1, 2, 3, 4):
                gi = [g for g in range(len(gbox)) if gtype[g] == t]
                pi = [p for p in range(len(pred)) if ptype[p] == t]
                iou = np.zeros((len(gi), len(pi)), np.float32)
                if gi and pi:
                    iou = boxes_iou3d(gbox[gi], pred[pi][:, :7]).astype(np.float32)
                    margin.add(iou[iou > 0], float(IOU_THRESH[t]), 'iou')
                valid = iou >= IOU_THRESH[t]
                per_type[t] = (gi, pi, iou, valid)
            pre.append((pred, pid, gbox, gobj, glevel, per_type))
        for t in (1, 2, 3, 4):
            for k in range(101):
                last_id, last_frame = {}, {}
                for f, (pred, pid, gbox, gobj, glevel, per_type) in enumerate(pre):
                    gi, pi, iou, valid = per_type[t]
                    active = [j for j in range(len(pi)) if pred[pi[j], 7] >= CUTOFFS[k]]
                    match = {}                                   # ground-truth position -> prediction position
                    for a in range(len(gi)):                      # 1. retention
                        o = gobj[gi[a]]
                        if last_frame.get(o) != f - 1:
                            continue
                        for j in active:
                            if pid[pi[j]] == last_id[o] and valid[a, j]:
                                match[a] = j
                    rows = [a for a in range(len(gi)) if a not in match]
                    taken = set(match.values())
                    cols = [j for j in active if j not in taken]
                    if rows and cols:                             # 2. fresh matching
                        w = np.where(valid[np.ix_(rows, cols)], iou[np.ix_(rows, cols)].astype(np.float64), 0.0)
                        r, c = linear_sum_assignment(w, maximize=True)
                        for i, j in zip(r, c):
                            if w[i, j] > 0:
                                match[rows[i]] = cols[j]
                    matched_preds = set(match.values())
                    for a, j in match.items():                    # 3. mismatches, counts
                        g, p = gi[a], pi[j]
                        o = gobj[g]
                        mis = o in last_id and last_id[o] != pid[p]
                        shards = [t - 1, 4 + 3 * (t - 1) + range_of(gbox[g])]
                        cost = int(np.rint((1.0 - float(iou[a, j])) * FIXED))
                        for lvl in (1, 2):
                            if (2 if glevel[g] == 2 else 1) <= lvl:
                                for s in shards:
                                    rec[s, lvl - 1, k] += [1, 0, 0, int(mis), cost]
                    for a in range(len(gi)):                      # misses
                        if a in match:
                            continue
                        g = gi[a]
                        for lvl in (1, 2):
                            if (2 if glevel[g] == 2 else 1) <= lvl:
                                for s in (t - 1, 4 + 3 * (t - 1) + range_of(gbox[g])):
                                    rec[s, lvl - 1, k, 1] += 1
                    for j in active:                              # FP
                        if j not in matched_preds:
                            for s in (t - 1, 4 + 3 * (t - 1) + range_of(pred[pi[j]])):
                                rec[s, :, k, 2] += 1
                    for a, j in match.items():                    # 4. state
                        o = gobj[gi[a]]
                        last_id[o], last_frame[o] = pid[pi[j]], f
    return rec, margin


def mot_dict(rec, breakdowns=('object',)):
    """{'OBJECT_TYPE_TYPE_VEHICLE_LEVEL_1/MOTA': [v], .../MOTP, /MISS, /MISMATCH, /FP, 'RANGE_TYPE_..._LEVEL_2/...': ...} at the
    cutoff of the largest MOTA (the lowest on a tie); 0 everywhere for a shard without counting ground truth"""
    out = {}
    shards = []
    if 'object' in breakdowns:
        shards += [(t, 'OBJECT_TYPE_TYPE_%s' % TYPE_NAMES[t]) for t in range(4)]
    if 'range' in breakdowns:
        shards += [(4 + 3 * t + r, 'RANGE_TYPE_%s_%s' % (TYPE_NAMES[t], RANGE_NAMES[r])) for t in range(4) for r in range(3)]
    for s, name in shards:
        for lvl in (0, 1):
            best = None
            for k in range(101):
                m, miss, fp, mm, cost = (int(v) for v in rec[s, lvl, k])
                n = m + miss
                if n == 0:
                    vals = (0.0, 0.0, 0.0, 0.0, 0.0)
                else:
                    vals = (1.0 - (miss + mm + fp) / n, cost / FIXED / m if m else 0.0, miss / n, mm / n, fp / n)
                if best is None or vals[0] > best[0]:
                    best = vals
            for key, v in zip(('MOTA', 'MOTP', 'MISS', 'MISMATCH', 'FP'), best):
                out['%s_LEVEL_%d/%s' % (name, lvl + 1, key)] = [v]
    return out


def prepare(prediction_infos, gt_infos, class_name, config_type=('object',), fake_gt_infos=True):
    """the sequences ``records`` takes, from the reference's frame dicts: prediction_infos per frame {'sequence_name', 'obj_ids',
    'boxes_lidar', 'score', 'name'}, gt_infos per frame {'sequence_name', 'annos': {'name', 'obj_ids', 'difficulty',
    'num_points_in_gt', 'gt_boxes_lidar'}}; frame i of both lists is the same frame.  Inputs are not modified."""
    for c in config_type:
        if c not in ('object', 'range'):
            raise ValueError('unknown config type %r' % (c,))
    assert len(prediction_infos) == len(gt_infos)
    if not len(gt_infos):
        return []
    pf, pb, ps, pt, pk, gf, gb, gt, gd, gk = [], [], [], [], [], [], [], [], [], []
    seq_of = []
    for i, (pinfo, info) in enumerate(zip(prediction_infos, gt_infos)):
        seq = info['sequence_name']
        seq_of.append(seq)
        n = len(pinfo['boxes_lidar'])
        ids = pinfo.get('obj_ids', np.zeros(0, np.int64)) if n == 0 else pinfo['obj_ids']
        if len(ids) != n:
            raise ValueError('frame %d: %d obj_ids for %d boxes' % (i, len(ids), n))
        pb.append(np.asarray(pinfo['boxes_lidar'])[:, :7].reshape(-1, 7))
        ps.append(np.asarray(pinfo['score']).reshape(-1))
        pt += [WAYMO_CLASSES.index(x) for x in pinfo['name']]
        pk += [(seq, pinfo['sequence_name'] + '-' + str(x)) for x in ids]
        pf.append(np.full(n, i))
        a = info['annos']
        names, npts = np.asarray(a['name']), np.asarray(a['num_points_in_gt'])
        diff = np.array(a['difficulty'], copy=True)
        zero = diff == 0
        diff[zero & (npts > 5)] = 1
        diff[zero & (npts <= 5)] = 2
        keep = np.array([x in class_name for x in names], bool) & (npts > 0)
        boxes = np.array(a['gt_boxes_lidar'])
        if fake_gt_infos:
            boxes = fakelidar_to_lidar(boxes)
        gb.append(boxes[keep][:, :7])
        gt += [WAYMO_CLASSES.index(x) for x in names[keep]]
        gd.append(diff[keep])
        gk += [(seq, x) for x in np.asarray(a['obj_ids'])[keep]]
        gf.append(np.full(int(keep.sum()), i))
    pf, pb, ps, pt = np.concatenate(pf), np.concatenate(pb, 0), np.concatenate(ps), np.array(pt, np.int64)
    gf, gb, gt, gd = np.concatenate(gf), np.concatenate(gb, 0), np.array(gt, np.int64), np.concatenate(gd)
    pb[:, -1] = limit_period(pb[:, -1], offset=0.5, period=np.pi * 2)
    gb[:, -1] = limit_period(gb[:, -1], offset=0.5, period=np.pi * 2)
    if ps.size and ps.max() > 1:
        ps = 1 / (1 + np.exp(-ps))
    index = {}                                                   # per sequence: key -> index in order of first appearance
    pid = np.array([index.setdefault(s, {}).setdefault(key, len(index[s])) for s, key in pk], np.int64)
    gindex = {}
    gobj = np.array([gindex.setdefault(s, {}).setdefault(key, len(gindex[s])) for s, key in gk], np.int64)
    order = list(dict.fromkeys(seq_of))
    out = []
    for seq in order:
        frames = []
        for i in [i for i, s in enumerate(seq_of) if s == seq]:
            p, g = pf == i, gf == i
            pred = np.zeros((int(p.sum()), 9), np.float32)
            pred[:, :7], pred[:, 7], pred[:, 8] = pb[p], ps[p], pt[p]
            frames.append((pred, pid[p], gb[g].astype(np.float32), gobj[g], gt[g], gd[g]))
        out.append(frames)
    return out


def waymo_evaluation(prediction_infos, gt_infos, class_name, config_type=('object',), distance_thresh=100, fake_gt_infos=True):
    seqs = prepare(prediction_infos, gt_infos, class_name, config_type, fake_gt_infos)
    breakdowns = tuple(c for c in ('object', 'range') if c in config_type)
    rec, margin = records(seqs)
    return mot_dict(rec, breakdowns), rec, margin

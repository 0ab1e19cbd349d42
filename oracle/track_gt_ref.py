"""numpy restatement of DetZero's two scorings of tracks against ground truth: the training-target assignment
(tracking/detzero_track/models/tracking_modules/target_assign.py:8-139) and the tracklet recall (tracking/detzero_track/utils/
track_recall.py:102-262 with get_trajectory_similarity / get_iou_mat_dict / get_gt_id_data of utils/track_calculation.py and
tracklets_to_frames of utils/data_utils.py).

Inputs are the reference's own forms: ``frames`` the frame dicts of one sequence in order (waymo_infos_<split>.pkl: 'sample_idx',
'pose', 'annos' with 'name', 'obj_ids', 'gt_boxes_lidar', 'gt_boxes_global', 'difficulty', 'num_points_in_gt'), ``tracks`` the
{track id: {'boxes_global', 'name', 'sample_idx', ...}} dict of one sequence (TrackResult.to_reference, sample_idx as frame-id
strings).  Frame ids are integers in ascending order, as get_trajectory_similarity walks them.

Arithmetic is that of the reference under numpy >= 2 (NEP 50), which is what the golden vectors (tests/golden/track_gt.npz) were
produced with: track boxes go to the lidar frame through the float32 inverse pose, IoUs are float32 and compared with the threshold as
float32, the per-pair sums accumulate in float32 in frame order, a similarity is the float32 quotient sum / trajectory length, and a
match rate is the float32 quotient match count / trajectory length compared with the float64 cutoffs np.arange(10) * 0.1.  So 3 of
10 frames (float32 0.3 = 0.30000001) passes the cutoff 0.30000000000000004; a float64 rate (0.29999999999999999) would not.

One deviation: where the reference raises TypeError in calculate_tracklet_recall (a difficulty and class with ground truth but no
matched trajectory, whose 'match_rate' list does not exist), tp is 0 here, as in detzero_b200.track.tracklet_recall.

``margin`` is the smallest distance from a decision over every compared value: each positive IoU against its class threshold, per
assignment component the cost gap to the best assignment that avoids one chosen edge (oracle.track_ref._assign), and each matched
object's first-to-last displacement against 1 m.  ``rate_margin`` is the smallest distance of a match rate from a cutoff; the device
forms the rates on the host from exact integer counts with this same arithmetic, so it bounds nothing and is reported only.
"""
from collections import defaultdict

import numpy as np

from . import boxes_iou3d, boxes_iou_bev
from .track_ref import CLASS_NAMES, Margin, _assign, yaw_filter

CUTOFFS = np.arange(0, 10) * 0.1


def lidar_boxes(boxes_global, pose):
    """transform_boxes3d(boxes, pose, inverse=True) of tracklets_to_frames: float32 boxes, float32 inverse pose, float64 centre
    product, float32 heading -> (n, 7) float32"""
    b = np.asarray(boxes_global, np.float32)[:, :7]
    inv = np.zeros((4, 4), np.float32)
    inv[:3, :3] = pose[:3, :3].T
    inv[:3, 3:] = -(pose[:3, :3].T @ pose[:3, 3:])
    inv[3, 3] = 1
    c = np.concatenate([b[:, :3], np.ones((len(b), 1))], -1) @ inv.T
    h = yaw_filter(b[:, [6]] + np.arctan2(inv[1, 0], inv[0, 0]))
    return np.concatenate([c[:, :3], b[:, 3:6], h], -1).astype(np.float32)


def _difficulty(d, n):
    d = np.array(d, copy=True)
    z = d == 0
    d[z & (np.asarray(n) > 5)] = 1
    d[z & (np.asarray(n) <= 5)] = 2
    return d


def score_sequence(frames, tracks, thresholds, recall, method='bev'):
    """The shared computation: per frame the class-masked IoU of the ground-truth rows of the classes in ``thresholds`` with the track
    boxes of that frame, per (object, track) the float32 sums and counts, the similarity matrix and the GNN assignment.
    Returns a dict: objects (ids in first-appearance order, with their rows), track ids, sim, count (match counts), pairs (the
    assignment), iou[(f, object, track)] (the IoU matrices' entries), and the margins."""
    margin, names = Margin(), list(thresholds)
    fids = [str(fr['sample_idx']) for fr in frames]
    fidx = {fid: f for f, fid in enumerate(fids)}
    tk_ids = list(tracks.keys())
    per_frame = defaultdict(list)                                  # frame -> [(track index, entry index)]
    for k, tid in enumerate(tk_ids):
        for j, sid in enumerate(tracks[tid]['sample_idx']):
            if str(sid) in fidx:
                per_frame[fidx[str(sid)]].append((k, j))
    obj_ids, objects = [], {}
    for f, fr in enumerate(frames):
        a = fr['annos']
        for g in range(len(a['name'])):
            if a['name'][g] not in names:
                continue
            oid = a['obj_ids'][g]
            if oid not in objects:
                objects[oid] = {'rows': [], 'index': len(obj_ids)}
                obj_ids.append(oid)
            objects[oid]['rows'].append((f, g))
    O, K = len(obj_ids), len(tk_ids)
    sums = np.zeros((O, K), np.float32)
    cnt = np.zeros((O, K), np.int64)
    ious = {}
    thr32 = {n: np.float32(t) for n, t in thresholds.items()}
    iou_fn = boxes_iou3d if method == '3d' else boxes_iou_bev
    for f, fr in enumerate(frames):
        a = fr['annos']
        rows = [g for g in range(len(a['name'])) if a['name'][g] in names]
        ent = sorted(per_frame[f], key=lambda kj: tk_ids[kj[0]])
        if not rows or not ent:
            continue
        gb = np.asarray(a['gt_boxes_lidar'], np.float32)[rows, :7]
        tb = np.concatenate([lidar_boxes(np.asarray(tracks[tk_ids[k]]['boxes_global'])[[j]], np.asarray(fr['pose'], np.float64))
                             for k, j in ent])
        m = iou_fn(gb, tb)
        for r, g in enumerate(rows):
            o = objects[a['obj_ids'][g]]['index']
            gn = a['name'][g]
            for i, (k, j) in enumerate(ent):
                v = m[r, i] if str(tracks[tk_ids[k]]['name'][j]) == gn else np.float32(0)
                if not v > 0:
                    continue
                ious[(f, o, k)] = v
                margin.add(v, thresholds[gn], 'iou')
                hit = v >= thr32[gn]
                if recall or hit:
                    sums[o, k] = sums[o, k] + v
                cnt[o, k] += int(hit)
    length = np.array([len(objects[oid]['rows']) for oid in obj_ids], np.int64)
    sim = np.full((O, K), -1, np.float32)
    ok = cnt > 0
    sim[ok] = (sums / np.maximum(length, 1).astype(np.float32)[:, None])[ok]
    pairs = _assign(ok, sim, margin, 'trajectory')
    return {'obj_ids': obj_ids, 'objects': objects, 'tk_ids': tk_ids, 'sim': sim, 'count': cnt, 'length': length,
            'pairs': pairs, 'ious': ious, 'margin': margin, 'fids': fids}


def assign_track_target(frames, tracks, iou_thresholds):
    """target_assign.assign_track_target of one sequence -> ({'label', 'unlabel'} as the reference returns it, margin).  'track'
    entries are the input track dicts plus 'iou' and, for a label, 'state'."""
    r = score_sequence(frames, tracks, iou_thresholds, recall=False, method='bev')
    margin = r['margin']
    label, unlabel = {}, {}
    matched = set()
    for o, k in r['pairs']:
        tid, oid = r['tk_ids'][k], r['obj_ids'][o]
        matched.add(k)
        t = dict(tracks[tid])
        t['iou'] = np.zeros(len(t['sample_idx']), np.float32)
        for j, sid in enumerate(t['sample_idx']):
            f = r['fids'].index(str(sid)) if str(sid) in r['fids'] else -1
            t['iou'][j] = r['ious'].get((f, o, k), np.float32(0))
        rows = r['objects'][oid]['rows']
        gt = {'gt_boxes_global': np.array([frames[f]['annos']['gt_boxes_global'][g] for f, g in rows]),
              'gt_boxes_lidar': np.array([frames[f]['annos']['gt_boxes_lidar'][g] for f, g in rows]),
              'name': np.array([frames[f]['annos']['name'][g] for f, g in rows]),
              'obj_ids': np.array([frames[f]['annos']['obj_ids'][g] for f, g in rows]),
              'sample_idx': np.array([r['fids'][f] for f, _ in rows])}
        d = float(np.linalg.norm(gt['gt_boxes_global'][0, :2] - gt['gt_boxes_global'][-1, :2], ord=2, axis=0))
        margin.add(d, 1.0, 'state')
        t['state'] = 'dynamic' if d > 1 else 'static'
        label[tid] = {'track': t, 'gt': gt}
    for k, tid in enumerate(r['tk_ids']):
        if k not in matched:
            unlabel[tid] = {'track': tracks[tid]}
    return {'label': label, 'unlabel': unlabel}, margin


def eval_single_seq(frames, tracks, class_names, iou_thresholds, method='3d', difficultys=('l1', 'l2')):
    """TrackRecall.eval_single_seq -> ({difficulty: {class: {'gt_box_nums_list', 'match_rate', 'match_pred_box_nums_list',
    'match_len', 'unmatch_pred_box_nums_list'}}}, margin, rate_margin)"""
    thr = dict(zip(class_names, iou_threshold_list(iou_thresholds, class_names)))
    r = score_sequence(frames, tracks, thr, recall=True, method=method)
    rate_margin = Margin()
    res = {d: {c: defaultdict(list) for c in class_names} for d in difficultys}
    diff = {}
    for oid in r['obj_ids']:
        rows = r['objects'][oid]['rows']
        diff[oid] = _difficulty([frames[f]['annos']['difficulty'][g] for f, g in rows],
                                [frames[f]['annos']['num_points_in_gt'][g] for f, g in rows])
    matched_o, matched_k = set(), set()
    for o, k in r['pairs']:
        oid = r['obj_ids'][o]
        f, g = r['objects'][oid]['rows'][0]
        name = frames[f]['annos']['name'][g]
        d = 'l2' if np.count_nonzero(diff[oid] == 2) > 0 else 'l1'
        n = len(diff[oid])
        rate = np.float32(r['count'][o, k]) / n
        rate_margin.add(np.full(len(CUTOFFS), rate, np.float64), CUTOFFS, 'match rate')
        res[d][name]['gt_box_nums_list'].append(n)
        res[d][name]['match_rate'].append(rate)
        res[d][name]['match_pred_box_nums_list'].append(len(tracks[r['tk_ids'][k]]['name']))
        res[d][name]['match_len'].append(np.float32(r['count'][o, k]))
        matched_o.add(o)
        matched_k.add(k)
    for k, tid in enumerate(r['tk_ids']):
        if k not in matched_k:
            for d in difficultys:
                res[d][str(tracks[tid]['name'][0])]['unmatch_pred_box_nums_list'].append(len(tracks[tid]['name']))
    for o, oid in enumerate(r['obj_ids']):
        if o not in matched_o:
            f, g = r['objects'][oid]['rows'][0]
            res[{1: 'l1', 2: 'l2'}[int(diff[oid][0])]][frames[f]['annos']['name'][g]]['gt_box_nums_list'].append(len(diff[oid]))
    return res, r['margin'], rate_margin


def iou_threshold_list(iou_thresholds, class_names):
    return [iou_thresholds[c] for c in class_names] if isinstance(iou_thresholds, dict) else list(iou_thresholds)


def calculate_tracklet_recall(eval_results, class_names, difficultys=('l1', 'l2')):
    """TrackRecall.calculate_tracklet_recall over the eval_single_seq results of several sequences"""
    out = {}
    for d in difficultys:
        out[d] = {}
        for c in class_names:
            lists = defaultdict(list)
            for e in eval_results:
                for key, v in e[d][c].items():
                    lists[key].extend(v)
            g = len(lists['gt_box_nums_list'])
            p = len(lists['match_pred_box_nums_list']) + len(lists['unmatch_pred_box_nums_list'])
            rates = np.array(lists['match_rate'])
            res = defaultdict(list)
            for cut in CUTOFFS:
                tp = np.count_nonzero(rates >= cut) if g > 0 and len(rates) else 0
                fp = p - tp
                res['precisions'].append(tp / (tp + fp + 1e-9))
                res['recalls'].append(tp / (g + 1e-9))
                res['tp'].append(tp)
                res['fp'].append(fp)
                res['pred_nums'].append(p)
                res['cutoffs'].append(float(cut))
                res['gt_nums'].append(g)
            out[d][c] = dict(res)
    return out


def tracklet_recall(sequences, class_names=CLASS_NAMES, iou_threshold=(0.7, 0.5, 0.5), method='3d'):
    """get_tracklet_recall over [(frames, tracks)] -> (table with 'iou_thresholds' and 'method', margin, rate_margin)"""
    margin, rate_margin, evals = Margin(), Margin(), []
    for frames, tracks in sequences:
        e, m, rm = eval_single_seq(frames, tracks, list(class_names), list(iou_threshold), method)
        evals.append(e)
        for a, b in ((margin, m), (rate_margin, rm)):
            if b.value < a.value:
                a.value, a.where = b.value, b.where
    out = calculate_tracklet_recall(evals, list(class_names))
    out['iou_thresholds'] = dict(zip(class_names, iou_threshold))
    out['method'] = method
    return out, margin, rate_margin

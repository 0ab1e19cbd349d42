"""Hand-computed cases of the tracking MOTA / MOTP metric (oracle/track_eval_ref.py, csrc/track_eval.cu): each case gives prepared
sequences (lists of frames (pred (n, 9) [box7, score, Waymo type], pred_id, gt_box (m, 7), gt_obj, gt_type, gt_level)), the
breakdowns, and a check of (records, metric dict)."""
import numpy as np

VEH = (4.0, 2.0, 1.5)


def box(x, y=0.0, h=0.0, size=VEH):
    return [x, y, 0.0, size[0], size[1], size[2], h]


def frame(preds, gts):
    """preds: [(box7, score, type, id)], gts: [(box7, type, level, object)]"""
    p = np.array([list(b) + [s, t] for b, s, t, _ in preds], np.float32).reshape(-1, 9)
    g = np.array([b for b, _, _, _ in gts], np.float32).reshape(-1, 7)
    return (p, np.array([i for _, _, _, i in preds], np.int64), g, np.array([o for _, _, _, o in gts], np.int64),
            np.array([t for _, t, _, _ in gts], np.int64), np.array([lv for _, _, lv, _ in gts], np.int64))


def pad_sequences(seqs):
    """prepared sequences -> the padded tables of evaluate.tracking_metrics (numpy)"""
    S = len(seqs)
    F = max([len(s) for s in seqs] + [1])
    R = max([len(f[0]) for s in seqs for f in s] + [1])
    G = max([len(f[2]) for s in seqs for f in s] + [1])
    t = {'pred': np.zeros((S, F, R, 9), np.float32), 'pred_id': np.zeros((S, F, R), np.int32), 'pred_cnt': np.zeros((S, F), np.int32),
         'gt_box': np.zeros((S, F, G, 7), np.float32), 'gt_obj': np.zeros((S, F, G), np.int32), 'gt_type': np.zeros((S, F, G), np.int32),
         'gt_level': np.zeros((S, F, G), np.int32), 'gt_cnt': np.zeros((S, F), np.int32), 'num_frames': np.zeros(S, np.int32),
         'n_obj': np.zeros(S, np.int32)}
    for s, frames in enumerate(seqs):
        t['num_frames'][s] = len(frames)
        for f, (p, pid, g, go, gt, gl) in enumerate(frames):
            t['pred'][s, f, :len(p)], t['pred_id'][s, f, :len(p)], t['pred_cnt'][s, f] = p, pid, len(p)
            t['gt_box'][s, f, :len(g)], t['gt_obj'][s, f, :len(g)], t['gt_cnt'][s, f] = g, go, len(g)
            t['gt_type'][s, f, :len(g)], t['gt_level'][s, f, :len(g)] = gt, gl
            if len(go):
                t['n_obj'][s] = max(t['n_obj'][s], int(np.max(go)) + 1)
    return t


def _close(a, b, tol=1e-12):
    assert abs(a - b) <= tol, (a, b)


def _veh(d, key, lvl=1):
    return d['OBJECT_TYPE_TYPE_VEHICLE_LEVEL_%d/%s' % (lvl, key)][0]


def _perfect():
    frames = [frame([(box(10.0 + f), 0.805, 1, 7), (box(-20.0, 5.0 - f), 0.805, 1, 3)],
                    [(box(10.0 + f), 1, 1, 0), (box(-20.0, 5.0 - f), 1, 1, 1)]) for f in range(3)]

    def check(rec, d):
        assert list(rec[0, 0, 80, :4]) == [6, 0, 0, 0] and list(rec[0, 0, 81, :4]) == [0, 6, 0, 0]
        _close(_veh(d, 'MOTA'), 1.0)
        assert _veh(d, 'MOTP') < 1e-6 and _veh(d, 'MISMATCH') == 0.0 and _veh(d, 'MISS') == 0.0
    return [frames], ('object',), check


def _id_switch():
    frames = [frame([(box(10.0), 0.9, 1, 1 if f < 2 else 2)], [(box(10.0), 1, 1, 0)]) for f in range(4)]

    def check(rec, d):
        assert list(rec[0, 0, 0, :4]) == [4, 0, 0, 1]
        _close(_veh(d, 'MOTA'), 0.75)
        _close(_veh(d, 'MISMATCH'), 0.25)
    return [frames], ('object',), check


def _retention():
    # pedestrian-sized thresholds (0.5) on vehicle-sized boxes: P1 overlaps G1 (0.907) and G2 (0.755), P2 overlaps G1 (0.951) and G2
    # (0.647), so the maximum IoU sum pairs P1-G2 and P2-G1.  In the second frame the predictions trade places: the IoU-sum optimum
    # (1.706) would swap both ids, but both previous pairs are still valid (1.554) and retention keeps them
    g1, g2 = box(0.0), box(0.8, size=(4.4, 2.0, 1.5))
    pa, pb = box(0.2, size=(4.2, 2.0, 1.5)), box(-0.1)
    gts = [(g1, 2, 1, 0), (g2, 2, 1, 1)]
    frames = [frame([(pa, 0.9, 2, 1), (pb, 0.9, 2, 2)], gts), frame([(pb, 0.9, 2, 1), (pa, 0.9, 2, 2)], gts)]

    def check(rec, d):
        assert list(rec[1, 0, 0, :4]) == [4, 0, 0, 0]
        _close(d['OBJECT_TYPE_TYPE_PEDESTRIAN_LEVEL_1/MOTA'][0], 1.0)
        # the frame-1 cost is that of the retained pairs, not of the IoU-sum optimum
        assert rec[1, 0, 0, 4] > round((2 * (2 - 1.706) + 0.07) * 2.0 ** 32)    # about 0.294 + 0.446, not 2 x 0.294
    return [frames], ('object',), check


def _gap():
    # object 0 keeps id 1 across a frame it is absent from (no mismatch); object 1 comes back with a new id (a mismatch)
    a, b = box(10.0), box(-10.0, 8.0)
    full = frame([(a, 0.9, 1, 1), (b, 0.9, 1, 2)], [(a, 1, 1, 0), (b, 1, 1, 1)])
    frames = [full, full, frame([], []), frame([(a, 0.9, 1, 1), (b, 0.9, 1, 3)], [(a, 1, 1, 0), (b, 1, 1, 1)])]

    def check(rec, d):
        assert list(rec[0, 0, 0, :4]) == [6, 0, 0, 1]
        _close(_veh(d, 'MISMATCH'), 1 / 6)
    return [frames], ('object',), check


def _level2():
    frames = [frame([(box(10.1), 0.7, 1, 4)], [(box(10.0), 1, 2, 0)]) for _ in range(2)]

    def check(rec, d):
        assert not rec[0, 0].any()                                        # neither a match nor an FP at LEVEL_1
        assert list(rec[0, 1, 0, :4]) == [2, 0, 0, 0] and list(rec[0, 1, 71, :4]) == [0, 2, 0, 0]
        assert all(_veh(d, k) == 0.0 for k in ('MOTA', 'MOTP', 'MISS', 'MISMATCH', 'FP'))
        _close(_veh(d, 'MOTA', 2), 1.0)
    return [frames], ('object',), check


def _low_score_fp():
    # an FP at score 0.305 in both frames: MOTA 0 up to cutoff 30, 1 from 31 to 90, so the lowest best cutoff is 31
    frames = [frame([(box(10.0), 0.905, 1, 1), (box(-30.0), 0.305, 1, 2)], [(box(10.0), 1, 1, 0)]) for _ in range(2)]

    def check(rec, d):
        assert list(rec[0, 0, 30, :4]) == [2, 0, 2, 0] and list(rec[0, 0, 31, :4]) == [2, 0, 0, 0]
        _close(_veh(d, 'MOTA'), 1.0)
        assert _veh(d, 'FP') == 0.0
    return [frames], ('object',), check


def _tie():
    # cutoffs 0..50: 2 matches and an FP; 51..90: 1 match and a miss; both MOTA 0.5, and the lowest cutoff (0) is reported
    frames = [frame([(box(10.0), 0.905, 1, 1), (box(-30.0), 0.505, 1, 2), (box(20.3, 5.0), 0.505, 1, 3)],
                    [(box(10.0), 1, 1, 0), (box(20.0, 5.0), 1, 1, 1)])]

    def check(rec, d):
        assert list(rec[0, 0, 50, :4]) == [2, 0, 1, 0] and list(rec[0, 0, 51, :4]) == [1, 1, 0, 0]
        _close(_veh(d, 'MOTA'), 0.5)
        _close(_veh(d, 'MISS'), 0.0)
        _close(_veh(d, 'FP'), 0.5)
        _close(_veh(d, 'MOTP'), rec[0, 0, 0, 4] / 2.0 ** 32 / 2)
    return [frames], ('object',), check


def _straddle():
    # one object crossing 30 m keeps its identity; its matches go to the range of the ground-truth box in each frame
    frames = [frame([(box(29.9), 0.9, 1, 5)], [(box(29.8), 1, 1, 0)]), frame([(box(30.2), 0.9, 1, 5)], [(box(30.1), 1, 1, 0)])]

    def check(rec, d):
        near, mid = 4, 5
        assert list(rec[near, 0, 0, :4]) == [1, 0, 0, 0] and list(rec[mid, 0, 0, :4]) == [1, 0, 0, 0]
        assert list(rec[0, 0, 0, :4]) == [2, 0, 0, 0]
        _close(d['RANGE_TYPE_VEHICLE_[30, 50)_LEVEL_1/MOTA'][0], 1.0)
    return [frames], ('object', 'range'), check


def _no_gt():
    frames = [frame([(box(5.0), 0.5, 2, 1)], []), frame([], [])]

    def check(rec, d):
        assert (rec[1, :, :51, 2] == 1).all() and (rec[4 + 3, :, :51, 2] == 1).all()
        rest = rec.copy()
        rest[1, :, :, 2] = rest[7, :, :, 2] = 0
        assert not rest.any()
        assert all(v == [0.0] for v in d.values()) and len(d) == 16 * 2 * 5
    return [frames], ('object', 'range'), check


CASES = {'perfect': _perfect, 'id_switch': _id_switch, 'retention': _retention, 'gap': _gap, 'level2': _level2,
         'low_score_fp': _low_score_fp, 'tie': _tie, 'straddle': _straddle, 'no_gt': _no_gt}

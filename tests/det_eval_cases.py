"""Hand-computed cases of the detection AP / APH metric (oracle/det_eval_ref.py, csrc/det_eval.cu): each case gives prepared frames
(pred (n, 9) [box7, score, Waymo type], gt_box (m, 7), gt_type, gt_level), the breakdowns, and a check of (records, ap dict)."""
import numpy as np

VEH = (4.0, 2.0, 1.5)


def box(x, y=0.0, h=0.0, size=VEH):
    return [x, y, 0.0, size[0], size[1], size[2], h]


def frame(preds, gts):
    """preds: [(box7, score, type)], gts: [(box7, type, level)]"""
    p = np.array([list(b) + [s, t] for b, s, t in preds], np.float32).reshape(-1, 9)
    g = np.array([b for b, _, _ in gts], np.float32).reshape(-1, 7)
    return (p, g, np.array([t for _, t, _ in gts], np.int64), np.array([lv for _, _, lv in gts], np.int64))


def pad_frames(frames):
    """prepared frames -> the padded tables of evaluate.detection_metrics (numpy)"""
    NF = len(frames)
    R = max([len(f[0]) for f in frames] + [1])
    G = max([len(f[1]) for f in frames] + [1])
    t = {'pred': np.zeros((NF, R, 9), np.float32), 'pred_cnt': np.zeros(NF, np.int32), 'gt_box': np.zeros((NF, G, 7), np.float32),
         'gt_type': np.zeros((NF, G), np.int32), 'gt_level': np.zeros((NF, G), np.int32), 'gt_cnt': np.zeros(NF, np.int32)}
    for i, (p, g, gt, gl) in enumerate(frames):
        t['pred'][i, :len(p)], t['pred_cnt'][i] = p, len(p)
        t['gt_box'][i, :len(g)], t['gt_type'][i, :len(g)], t['gt_level'][i, :len(g)], t['gt_cnt'][i] = g, gt, gl, len(g)
    return t


def _close(a, b, tol=1e-12):
    assert abs(a - b) <= tol, (a, b)


def _perfect():
    gts = [(box(10.0), 1, 1), (box(35.0, h=0.4), 1, 1), (box(-60.0, h=-2.0), 1, 1)]
    preds = [(b, 0.805 + 0.01 * i, 1) for i, (b, _, _) in enumerate(gts)]

    def check(rec, ap):
        for lvl in (1, 2):
            _close(ap['OBJECT_TYPE_TYPE_VEHICLE_LEVEL_%d/AP' % lvl][0], 1.0)
            _close(ap['OBJECT_TYPE_TYPE_VEHICLE_LEVEL_%d/APH' % lvl][0], 1.0)
            for r in ('[0, 30)', '[30, 50)', '[50, +inf)'):
                _close(ap['RANGE_TYPE_VEHICLE_%s_LEVEL_%d/AP' % (r, lvl)][0], 1.0)
            _close(ap['OBJECT_TYPE_TYPE_SIGN_LEVEL_%d/AP' % lvl][0], 0.0)
        assert list(rec[0, 0, 80]) == [3, 0, 0, 3 << 32] and list(rec[0, 0, 81]) == [2, 0, 1, 2 << 32]
    return [frame(preds, gts)], ('object', 'range'), check


def _flipped():
    gts = [(box(10.0), 1, 1), (box(20.0, 5.0, h=1.0), 1, 1)]
    preds = [(box(10.0, h=np.pi), 0.6, 1), (box(20.0, 5.0, h=1.0 - np.pi), 0.7, 1)]

    def check(rec, ap):
        _close(ap['OBJECT_TYPE_TYPE_VEHICLE_LEVEL_1/AP'][0], 1.0)
        _close(ap['OBJECT_TYPE_TYPE_VEHICLE_LEVEL_1/APH'][0], 0.0, 1e-6)
    return [frame(preds, gts)], ('object',), check


def _false_positives():
    gts = [(box(10.0), 1, 1)]
    preds = [(box(-10.0), 0.9, 1), (box(10.0, 10.0), 0.5, 1), (box(10.0), 0.8, 2)]   # elsewhere, or of another type

    def check(rec, ap):
        _close(ap['OBJECT_TYPE_TYPE_VEHICLE_LEVEL_1/AP'][0], 0.0)
        _close(ap['OBJECT_TYPE_TYPE_PEDESTRIAN_LEVEL_1/AP'][0], 0.0)
        assert list(rec[0, 0, 0]) == [0, 2, 1, 0] and list(rec[1, 1, 0]) == [0, 1, 0, 0]
    return [frame(preds, gts)], ('object',), check


def _level2():
    gts = [(box(10.0), 1, 2)]
    preds = [(box(10.1), 0.7, 1)]

    def check(rec, ap):
        assert list(rec[0, 0, 0]) == [0, 0, 0, 0] and list(rec[0, 0, 70]) == [0, 0, 0, 0]
        assert rec[0, 1, 70, 0] == 1 and rec[0, 1, 70, 1] == 0 and rec[0, 1, 71, 2] == 1
        _close(ap['OBJECT_TYPE_TYPE_VEHICLE_LEVEL_1/AP'][0], 0.0)
        _close(ap['OBJECT_TYPE_TYPE_VEHICLE_LEVEL_2/AP'][0], 1.0)
    return [frame(preds, gts)], ('object',), check


def _range_boundary():
    gts = [(box(30.1), 1, 1)]
    preds = [(box(29.9), 0.6, 1)]

    def check(rec, ap):
        near, mid = 4, 5                      # vehicle [0, 30), [30, 50)
        assert list(rec[mid, 0, 60, :3]) == [1, 0, 0] and list(rec[near, 0, 60]) == [0, 0, 0, 0]
        assert list(rec[near, 0, 0]) == [0, 0, 0, 0]
        _close(ap['RANGE_TYPE_VEHICLE_[30, 50)_LEVEL_1/AP'][0], 1.0)
    return [frame(preds, gts)], ('object', 'range'), check


def _score_half():
    gts = [(box(10.0), 1, 1)]
    preds = [(box(10.0), 0.5, 1)]

    def check(rec, ap):
        assert list(rec[0, 0, 50, :3]) == [1, 0, 0] and list(rec[0, 0, 51, :3]) == [0, 0, 1]
    return [frame(preds, gts)], ('object',), check


def _contention():
    # P1 overlaps G1 (0.907) and G2 (0.755), P2 only G1 (0.951; 0.647 with G2): the maximum IoU sum pairs P1-G2 and P2-G1
    g1, g2 = box(0.0), box(0.8, size=(4.4, 2.0, 1.5))
    p1, p2 = box(0.2, size=(4.2, 2.0, 1.5)), box(-0.1)
    gts = [(g1, 1, 1), (g2, 1, 1)]
    preds = [(p1, 0.9, 1), (p2, 0.4, 1)]
    # a second frame: two predictions on one object, the better one with the lower score
    gts2 = [(box(50.0, 5.0), 1, 1)]
    preds2 = [(box(50.3, 5.0), 0.9, 1), (box(50.1, 5.0), 0.6, 1)]

    def check(rec, ap):
        assert list(rec[0, 0, 40, :3]) == [3, 1, 0]            # both pairs of frame 1, the better of frame 2, its duplicate FP
        assert list(rec[0, 0, 41, :3]) == [2, 1, 1]            # P2 inactive: P1 takes G1; frame 2 unchanged
        assert list(rec[0, 0, 61, :3]) == [2, 0, 1]            # frame 2: only the worse prediction is left, and matches
    return [frame(preds, gts), frame(preds2, gts2)], ('object',), check


def _envelope():
    gts = [(box(10.0), 1, 1), (box(20.0), 1, 1), (box(30.0, 10.0), 1, 1)]
    preds = [(box(10.0), 0.905, 1), (box(-20.0), 0.805, 1), (box(20.0), 0.705, 1), (box(30.0, 10.0), 0.305, 1)]

    def check(rec, ap):
        # points: r 1/3 p 1 (k 81..90), r 1/3 p 1/2 (71..80), r 2/3 p 2/3 (31..70), r 1 p 3/4 (0..30): 1/3 + 1/3 * 3/4 + 1/3 * 3/4
        _close(ap['OBJECT_TYPE_TYPE_VEHICLE_LEVEL_1/AP'][0], 1 / 3 + 0.5, 1e-12)
    return [frame(preds, gts)], ('object',), check


def _empty():
    # an empty frame, and a sign without any prediction: FN of the sign shards, nothing else
    def check(rec, ap):
        assert (rec[2, :, :, 2] == 1).all() and (rec[10, :, :, 2] == 1).all()
        rest = rec.copy()
        rest[2, :, :, 2] = rest[10, :, :, 2] = 0
        assert not rest.any()
        assert all(v == [0.0] for v in ap.values()) and len(ap) == 2 * 2 * 16
    return [frame([], []), frame([], [(box(5.0, size=(0.5, 0.5, 2.0)), 3, 1)])], ('object', 'range'), check


CASES = {'perfect': _perfect, 'flipped': _flipped, 'false_positives': _false_positives, 'level2': _level2,
         'range_boundary': _range_boundary, 'score_half': _score_half, 'contention': _contention, 'envelope': _envelope,
         'empty': _empty}

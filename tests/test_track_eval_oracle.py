"""The numpy restatement of the tracking MOTA / MOTP metric (oracle/track_eval_ref.py) on hand-computed cases, the metric dict's
keys, and the host preparation of the reference-shaped entry point (oracle/track_eval_ref.prepare and
detzero_b200.evaluate.tracking_tables, which must agree)."""
import numpy as np
import pytest

from detzero_b200 import evaluate
from oracle import track_eval_ref
from tests import track_eval_cases


@pytest.mark.parametrize('name', sorted(track_eval_cases.CASES))
def test_hand_case(name):
    seqs, breakdowns, check = track_eval_cases.CASES[name]()
    rec, margin = track_eval_ref.records(seqs)
    d = track_eval_ref.mot_dict(rec, breakdowns)
    check(rec, d)
    assert evaluate.mot_dict(rec, breakdowns) == d


def test_mot_dict_keys():
    rec = np.zeros((16, 2, 101, 5), np.int64)
    d = evaluate.mot_dict(rec, ('object', 'range'))
    types = ('VEHICLE', 'PEDESTRIAN', 'SIGN', 'CYCLIST')
    want = {'OBJECT_TYPE_TYPE_%s_LEVEL_%d/%s' % (t, l, m) for t in types for l in (1, 2) for m in evaluate.MOT_KEYS}
    want |= {'RANGE_TYPE_%s_%s_LEVEL_%d/%s' % (t, r, l, m) for t in types for r in ('[0, 30)', '[30, 50)', '[50, +inf)')
             for l in (1, 2) for m in evaluate.MOT_KEYS}
    assert set(d) == want and all(v == [0.0] for v in d.values())
    assert set(evaluate.mot_dict(rec, ('object',))) == {k for k in want if k.startswith('OBJECT')}


def _infos(seq, pred_rows, gt_rows, ids=None):
    """one frame: pred_rows [(box7, score, name, obj_id)], gt_rows [(box7, name, difficulty, num_points, obj_id)]"""
    p = {'sequence_name': seq, 'boxes_lidar': np.array([r[0] for r in pred_rows], np.float32).reshape(-1, 7),
         'score': np.array([r[1] for r in pred_rows], np.float32), 'name': np.array([r[2] for r in pred_rows]),
         'obj_ids': np.array([r[3] for r in pred_rows] if ids is None else ids, np.int64)}
    a = {'gt_boxes_lidar': np.array([r[0] for r in gt_rows], np.float32).reshape(-1, 7), 'name': np.array([r[1] for r in gt_rows]),
         'difficulty': np.array([r[2] for r in gt_rows], np.int32), 'num_points_in_gt': np.array([r[3] for r in gt_rows], np.int32),
         'obj_ids': np.array([r[4] for r in gt_rows])}
    return p, {'sequence_name': seq, 'annos': a}


def _both(preds, gts, class_name=('Vehicle', 'Pedestrian', 'Cyclist'), fake_gt_infos=False):
    """oracle sequences and evaluate.tracking_tables of the same infos; checks that they agree"""
    seqs = track_eval_ref.prepare(preds, gts, list(class_name), ('object',), fake_gt_infos)
    t = evaluate.tracking_tables(preds, gts, list(class_name), fake_gt_infos)
    want = track_eval_cases.pad_sequences(seqs)
    for k in want:
        got = t[k]
        if got.ndim == 4:
            got = got[:, :, :want[k].shape[2]]
        elif got.ndim == 3:
            got = got[:, :, :want[k].shape[2]]
        np.testing.assert_array_equal(got, want[k], err_msg=k)
    return seqs, t


def test_prepare_interleaved_sequences():
    b = track_eval_cases.box
    frames = [_infos('A', [(b(5.0), 0.5, 'Vehicle', 11)], [(b(5.0), 'Vehicle', 0, 10, 'a0')]),
              _infos('B', [(b(7.0), 0.6, 'Cyclist', 11), (b(9.0), 0.6, 'Sign', 12)], [(b(7.0), 'Cyclist', 0, 3, 'b0')]),
              _infos('A', [(b(6.0), 0.5, 'Vehicle', 12), (b(5.5), 0.5, 'Vehicle', 11)],
                     [(b(6.0), 'Vehicle', 2, 10, 'a1'), (b(5.5), 'Vehicle', 0, 10, 'a0')]),
              _infos('B', [], [(b(8.0), 'Cyclist', 0, 9, 'b0')])]
    preds, gts = [f[0] for f in frames], [f[1] for f in frames]
    seqs, t = _both(preds, gts)
    assert t['sequences'] == ['A', 'B'] and list(t['num_frames']) == [2, 2] and list(t['n_obj']) == [2, 1]
    assert [list(f[1]) for f in seqs[0]] == [[0], [1, 0]] and [list(f[1]) for f in seqs[1]] == [[0, 1], []]
    assert list(seqs[1][0][0][:, 8]) == [4, 3]                      # Cyclist 4, Sign 3 (the tracking evaluator's classes)
    assert list(seqs[0][1][5]) == [2, 1] and list(seqs[1][0][5]) == [2]   # difficulty 0 -> 1 / 2 by the point count
    assert list(gts[0]['annos']['difficulty']) == [0]                # the input is not modified


def test_prepare_class_filter_and_points():
    b = track_eval_cases.box
    p, g = _infos('A', [], [(b(5.0), 'Vehicle', 1, 6, 'v'), (b(10.0), 'Sign', 1, 5, 's'), (b(15.0), 'Vehicle', 1, 0, 'z'),
                            (b(20.0), 'Pedestrian', 1, 4, 'p')])
    seqs, _ = _both([p], [g], class_name=('Vehicle', 'Pedestrian'))
    _, _, gbox, gobj, gtype, _ = seqs[0][0]
    assert list(gbox[:, 0]) == [5.0, 20.0] and list(gtype) == [1, 2] and list(gobj) == [0, 1]


def test_prepare_sigmoid_and_heading():
    b = track_eval_cases.box
    p, g = _infos('A', [(b(5.0, h=4.0), 0.0, 'Vehicle', 1), (b(7.0), 2.0, 'Vehicle', 2)], [])
    seqs, _ = _both([p], [g])
    pred = seqs[0][0][0]
    assert pred[0, 7] == np.float32(0.5) and abs(pred[1, 7] - 1 / (1 + np.exp(-2.0))) < 1e-7
    assert abs(pred[0, 6] - (4.0 - 2 * np.pi)) < 1e-6
    p2, g2 = _infos('A', [(b(5.0), 1.0, 'Vehicle', 1)], [])
    assert _both([p2], [g2])[0][0][0][0][0, 7] == 1.0               # a maximum of 1: no sigmoid


def test_prepare_fake_lidar():
    p, g = _infos('A', [], [([1.0, 2.0, 3.0, 2.0, 4.0, 1.5, 0.25], 'Vehicle', 1, 10, 'v')])
    seqs, _ = _both([p], [g], fake_gt_infos=True)
    np.testing.assert_allclose(seqs[0][0][2][0], [1.0, 2.0, 3.75, 4.0, 2.0, 1.5, -(0.25 + np.pi / 2)], rtol=0, atol=1e-6)
    assert g['annos']['gt_boxes_lidar'][0, 2] == 3.0


def test_prepare_misaligned_ids_raise():
    b = track_eval_cases.box
    p, g = _infos('A', [(b(5.0), 0.5, 'Vehicle', 1), (b(9.0), 0.5, 'Vehicle', 2)], [], ids=[1])
    with pytest.raises(ValueError, match='obj_ids'):
        evaluate.tracking_tables([p], [g], ['Vehicle'])
    with pytest.raises(ValueError):
        track_eval_ref.prepare([p], [g], ['Vehicle'])


def test_unknown_config_type_and_name():
    b = track_eval_cases.box
    p, g = _infos('A', [(b(5.0), 0.5, 'Truck', 1)], [])
    with pytest.raises(ValueError, match='config type'):
        evaluate.WaymoTrackingMetricsEstimator().waymo_evaluation([p], [g], ['Vehicle'], config_type=['object', '3d'])
    with pytest.raises(ValueError):
        evaluate.tracking_tables([p], [g], ['Vehicle'])


def test_duplicate_ids_raise_in_oracle():
    seqs = [[track_eval_cases.frame([(track_eval_cases.box(5.0), 0.5, 1, 3), (track_eval_cases.box(-5.0), 0.5, 2, 3)], [])]]
    with pytest.raises(ValueError, match='share'):
        track_eval_ref.records(seqs)

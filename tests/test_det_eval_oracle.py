"""The numpy restatement of the detection AP / APH metric (oracle/det_eval_ref.py) on hand-computed cases, and the host preparation
of the reference-shaped entry point (oracle/det_eval_ref.prepare and detzero_b200.evaluate.frame_tables, which must agree)."""
import numpy as np
import pytest

from detzero_b200 import evaluate
from oracle import det_eval_ref
from tests import det_eval_cases


@pytest.mark.parametrize('name', sorted(det_eval_cases.CASES))
def test_hand_case(name):
    frames, breakdowns, check = det_eval_cases.CASES[name]()
    rec, _ = det_eval_ref.records(frames, '3d', breakdowns)
    check(rec, det_eval_ref.ap_dict(rec, breakdowns))
    rec_bev, _ = det_eval_ref.records(frames, 'bev', breakdowns)
    check(rec_bev, det_eval_ref.ap_dict(rec_bev, breakdowns))


def test_no_frames():
    rec, _ = det_eval_ref.records([], '3d', ('object',))
    assert rec.shape == (16, 2, 101, 4) and not rec.any()
    ap = det_eval_ref.ap_dict(rec, ('object',))
    assert sorted(ap) == sorted('OBJECT_TYPE_TYPE_%s_LEVEL_%d/%s' % (t, l, m) for t in det_eval_ref.TYPE_NAMES for l in (1, 2)
                                for m in ('AP', 'APH'))


def test_envelope_integral():
    # recall 0.5 at precision 0.4 and 1.0, recall 1.0 at precision 0.6: the envelope lifts the first point to 1.0
    tp, fp, fn = np.array([2, 1, 1, 0]), np.array([1, 0, 1.5, 0]), np.array([0, 1, 1, 2])
    want = 0.5 * 1.0 + 0.5 * (2 / 3)
    assert abs(det_eval_ref.average_precision(tp, fp, fn) - want) < 1e-15
    assert evaluate.average_precision(tp, fp, fn) == det_eval_ref.average_precision(tp, fp, fn)


def _infos(pred_rows, gt_rows):
    """one frame: pred_rows [(box7, score, name)], gt_rows [(box7, name, difficulty, num_points)]"""
    p = {'boxes_lidar': np.array([r[0] for r in pred_rows], np.float32).reshape(-1, 7),
         'score': np.array([r[1] for r in pred_rows], np.float32), 'name': np.array([r[2] for r in pred_rows])}
    g = {'gt_boxes_lidar': np.array([r[0] for r in gt_rows], np.float32).reshape(-1, 7), 'name': np.array([r[1] for r in gt_rows]),
         'difficulty': np.array([r[2] for r in gt_rows], np.int32), 'num_points_in_gt': np.array([r[3] for r in gt_rows], np.int32)}
    return p, g


def _both(preds, gts, **kw):
    """oracle frames and evaluate.frame_tables of the same infos; checks that they agree"""
    args = dict(class_name=['Vehicle', 'Pedestrian', 'Cyclist'], distance_thresh=100, fake_gt_infos=False)
    args.update(kw)
    frames = det_eval_ref.prepare(preds, gts, args['class_name'], ('object',), args['distance_thresh'], args['fake_gt_infos'])
    t = evaluate.frame_tables(preds, gts, **args)
    want = det_eval_cases.pad_frames(frames)
    for k in want:
        np.testing.assert_array_equal(t[k][:, :want[k].shape[1]] if t[k].ndim > 1 else t[k], want[k], err_msg=k)
    return frames


def test_prepare_difficulty_and_points():
    b = det_eval_cases.box
    p, g = _infos([], [(b(5.0), 'Vehicle', 0, 6), (b(10.0), 'Vehicle', 0, 5), (b(15.0), 'Vehicle', 0, 0), (b(20.0), 'Vehicle', 2, 100),
                       (b(25.0), 'Sign', 0, 50), (b(30.0), 'Pedestrian', 1, 1)])
    frames = _both([p], [g])
    _, gbox, gtype, glevel = frames[0]
    assert list(gbox[:, 0]) == [5.0, 10.0, 20.0, 30.0]          # no points, or a class not evaluated: dropped
    assert list(gtype) == [1, 1, 1, 2] and list(glevel) == [1, 2, 2, 1]
    assert list(g['difficulty']) == [0, 0, 0, 2, 0, 1]         # the input is not modified


def test_prepare_distance_boundary_and_heading():
    b = det_eval_cases.box
    p, g = _infos([(b(100.49, h=4.0), 0.5, 'Vehicle'), (b(100.5), 0.5, 'Cyclist'), (b(0.0, -100.4), 0.5, 'Truck')],
                  [(b(100.51), 'Vehicle', 1, 10), (b(60.0, 80.0), 'Vehicle', 1, 10), (b(59.9, 80.0), 'Cyclist', 1, 10)])
    frames = _both([p], [g])
    pred, gbox, gtype, _ = frames[0]
    assert list(pred[:, 0]) == [np.float32(100.49), 0.0] and list(pred[:, 8]) == [1, 3]
    assert abs(pred[0, 6] - (4.0 - 2 * np.pi)) < 1e-6           # limit_period(h, 0.5, 2 pi)
    assert list(gbox[:, 0]) == [60.0, np.float32(59.9)] and list(gtype) == [1, 4]     # kept where ||(x, y)|| < 100 + 0.5
    assert det_eval_ref.range_of(gbox[1]) == 2


def test_prepare_sigmoid_branch():
    b = det_eval_cases.box
    p1, g1 = _infos([(b(5.0), 0.5, 'Vehicle'), (b(7.0), 1.0, 'Vehicle')], [])
    assert list(_both([p1], [g1])[0][0][:, 7]) == [0.5, 1.0]              # maximum 1: no sigmoid
    p2, g2 = _infos([(b(5.0), 0.0, 'Vehicle'), (b(7.0), 2.0, 'Vehicle'), (b(900.0), 50.0, 'Vehicle')], [])
    s = _both([p2], [g2])[0][0][:, 7]
    assert s[0] == np.float32(0.5) and abs(s[1] - 1 / (1 + np.exp(-2.0))) < 1e-7


def test_prepare_fake_lidar():
    p, g = _infos([], [([1.0, 2.0, 3.0, 2.0, 4.0, 1.5, 0.25], 'Vehicle', 1, 10)])
    frames = _both([p], [g], fake_gt_infos=True)
    np.testing.assert_allclose(frames[0][1][0], [1.0, 2.0, 3.75, 4.0, 2.0, 1.5, -(0.25 + np.pi / 2)], rtol=0, atol=1e-6)
    assert g['gt_boxes_lidar'][0, 2] == 3.0


def test_unknown_config_type():
    p, g = _infos([], [])
    with pytest.raises(ValueError, match='config type'):
        det_eval_ref.prepare([p], [g], ['Vehicle'], ('object', 'iou'))
    with pytest.raises(ValueError, match='config type'):
        evaluate.WaymoDetectionMetricsEstimator().waymo_evaluation([p], [g], ['Vehicle'], config_type=['object', 'iou'])

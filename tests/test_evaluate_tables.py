"""The tables detzero_b200.evaluate builds before a metric call, on hand cases (CPU tensors, no kernel): which rows the distance cut,
the sigmoid's maximum and the prediction count of each entry point see."""
import numpy as np
import torch

from detzero_b200 import evaluate
from detzero_b200.offboard import OffboardResult
from detzero_b200.track import CLASS_NAMES, ground_truth_from_infos


def _box(x):
    return [x, 0.0, 0.0, 4.0, 2.0, 1.5, 0.0]


def _gt(rows):
    """a GroundTruth of one sequence of one frame: rows [(x, name, obj_id)], 10 points each, difficulty 1"""
    a = {'name': np.array([r[1] for r in rows]), 'obj_ids': np.array([r[2] for r in rows]),
         'gt_boxes_lidar': np.array([_box(r[0]) for r in rows], np.float32), 'gt_boxes_global': np.zeros((len(rows), 9)),
         'difficulty': np.ones(len(rows), np.int32), 'num_points_in_gt': np.full(len(rows), 10, np.int32)}
    return ground_truth_from_infos([{'sequence_name': 's', 'frame_id': 0, 'pose': np.eye(4), 'annos': a}], ['s'], device='cpu')


def _result(rows, obj_id, count):
    """an OffboardResult of one frame: rows [(x, score, label)]"""
    r = torch.tensor([[*_box(x), s, c] for x, s, c in rows], dtype=torch.float32)[None]
    return OffboardResult({}, None, r, torch.tensor([obj_id], dtype=torch.int32), torch.tensor([count], dtype=torch.int32))


def test_offboard_out_of_range_prediction():
    """a prediction beyond distance_thresh + 0.5 keeps its box but gets type 0, and its score does not select the sigmoid"""
    gt = _gt([(5.0, 'Vehicle', 'a')])
    res = _result([(5.0, 0.75, 1), (20.0, 0.5, 3), (150.0, 4.0, 2)], [0, 1, 2], 3)
    t = evaluate._offboard_tables([res], gt, CLASS_NAMES, 100)
    assert t['pred_cnt'].tolist() == [3] and t['pred'][0, 2, 0] == 150.0
    assert t['pred'][0, :, 7].tolist() == [0.75, 0.5, 4.0]
    assert t['pred'][0, :, 8].tolist() == [1, 4, 0]
    t = evaluate._offboard_tables([res], gt, CLASS_NAMES, 200)
    np.testing.assert_allclose(t['pred'][0, :, 7], 1 / (1 + np.exp(-np.array([0.75, 0.5, 4.0]))), rtol=1e-6)
    assert t['pred'][0, :, 8].tolist() == [1, 4, 2]


def test_frame_tables_sigmoid_after_distance_cut():
    p = {'boxes_lidar': np.array([_box(5.0), _box(150.0)], np.float32), 'score': np.array([0.75, 4.0], np.float32),
         'name': np.array(['Vehicle', 'Vehicle'])}
    g = {'gt_boxes_lidar': np.zeros((0, 7), np.float32), 'name': np.array([]), 'difficulty': np.zeros(0, np.int32),
         'num_points_in_gt': np.zeros(0, np.int32)}
    t = evaluate.frame_tables([p], [g], CLASS_NAMES, 100, False)
    assert t['pred_cnt'].tolist() == [1] and t['pred'][0, 0, 7] == np.float32(0.75)


def test_far_ground_truth_cut_for_detection_only():
    gt = _gt([(5.0, 'Vehicle', 'a'), (150.0, 'Pedestrian', 'b'), (20.0, 'Cyclist', 'c'), (30.0, 'Sign', 'd')])
    res = _result([(5.0, 0.5, 1)], [0], 1)
    det = evaluate._offboard_tables([res], gt, CLASS_NAMES, 100)
    assert det['gt_type'].tolist() == [[1, 0, 4, 0]] and det['gt_cnt'].tolist() == [4] and det['gt_box'][0, 1, 0] == 150.0
    trk = evaluate._offboard_tracking_tables([res], gt, CLASS_NAMES)
    assert trk['gt_type'].tolist() == [[[1, 2, 4, 0]]] and trk['gt_obj'].tolist() == [[[0, 1, 2, -1]]]


def test_offboard_tracking_counts_track_rows_only():
    """dropped detections (obj_id -1) follow the track rows; neither they nor rows past the count are predictions, and their scores
    do not select the sigmoid.  The detection tables count every live row."""
    gt = _gt([(5.0, 'Vehicle', 'a')])
    res = _result([(5.0, 0.9, 1), (9.0, 0.8, 2), (40.0, 3.0, 1), (60.0, 0.7, 3), (80.0, 5.0, 1)], [4, 7, -1, -1, 9], 4)
    t = evaluate._offboard_tracking_tables([res], gt, CLASS_NAMES)
    assert t['pred_cnt'].tolist() == [[2]] and t['pred_id'].tolist() == [[[4, 7, -1, -1, 9]]]
    assert t['pred'][0, 0, :, 7].tolist() == [np.float32(x) for x in (0.9, 0.8, 3.0, 0.7, 5.0)]
    assert t['pred'][0, 0, :, 8].tolist() == [1, 2, 0, 0, 0]
    det = evaluate._offboard_tables([res], gt, CLASS_NAMES, 1000)
    assert det['pred_cnt'].tolist() == [4] and det['pred'][0, :, 8].tolist() == [1, 2, 1, 4, 0]
    np.testing.assert_allclose(det['pred'][0, :4, 7], 1 / (1 + np.exp(-np.array([0.9, 0.8, 3.0, 0.7]))), rtol=1e-6)

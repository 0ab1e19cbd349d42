"""oracle/track_gt_ref.py (the numpy restatement of DetZero's target assignment and tracklet recall) against the golden vectors the
reference's own target_assign.assign_track_target and TrackRecall produced (tests/golden/make_golden_track_gt.py)."""
import numpy as np

from oracle import track_gt_ref
from tests import track_gt_golden

THR = {'Vehicle': 0.3, 'Pedestrian': 0.1, 'Cyclist': 0.1}


def test_assign_equals_golden():
    g, frames, tracks = track_gt_golden.load()
    out, margin = track_gt_ref.assign_track_target(frames, tracks, THR)
    assert list(out['label']) == g['label_tk'].tolist()
    assert list(out['unlabel']) == g['unlabel_tk'].tolist()
    assert [v['gt']['obj_ids'][0] for v in out['label'].values()] == g['label_obj'].tolist()
    assert [v['track']['state'] == 'dynamic' for v in out['label'].values()] == g['label_state'].tolist()
    assert np.array_equal(np.concatenate([v['track']['iou'] for v in out['label'].values()]), g['label_iou'])
    assert np.array_equal(np.concatenate([v['gt']['sample_idx'] for v in out['label'].values()]), g['label_gt_sample_idx'])
    assert margin.value >= 1e-3, (margin.value, margin.where)


def test_tracklet_recall_equals_golden():
    g, frames, tracks = track_gt_golden.load()
    table, margin, rate_margin = track_gt_ref.tracklet_recall([(frames, tracks)])
    ref = track_gt_golden.recall_table(g)
    for d in ('l1', 'l2'):
        for c in track_gt_golden.CLASS_NAMES:
            for k, v in ref[d][c].items():
                assert np.array_equal(np.asarray(table[d][c][k]), v), (d, c, k)
    assert table['method'] == '3d' and table['iou_thresholds'] == {'Vehicle': 0.7, 'Pedestrian': 0.5, 'Cyclist': 0.5}
    assert margin.value >= 1e-3, (margin.value, margin.where)
    assert rate_margin.value < 1e-6                       # the scene has a match rate on a cutoff (3 of 10 frames)


def test_match_rate_on_the_cutoff_is_float32():
    # 3 / 10 as float32 passes the float64 cutoff 3 * 0.1; as float64 it would not
    assert np.float32(3) / 10 >= track_gt_ref.CUTOFFS[3]
    assert not (3 / 10 >= track_gt_ref.CUTOFFS[3])

"""The numpy restatement of the DetZero tracker (oracle/track_ref.py) against tests/golden/track.npz, the output of the reference's
own DataProcessor, TrackManager and PostProcessor (tests/golden/make_golden_track.py), and the oracle's decision margin."""
import os

import numpy as np

from detzero_b200 import synthetic
from detzero_b200.track import tracker_cfg
from oracle import track_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'track.npz')


def test_oracle_matches_reference_golden():
    g = np.load(GOLDEN)
    r = track_ref.track_sequence(g['boxes'], g['counts'], g['poses'], tracker_cfg())
    assert r['margin'].value >= 1e-3, (r['margin'].value, r['margin'].where)
    for f, k in enumerate(r['kept']):
        assert np.array_equal(k, g['kept'][f, :len(k)]), f
    assert (~g['kept']).sum() >= 3
    assert set(g['trk'][:, 1]) == {1, 2, 3}
    assert [int(t[0]) for t in g['trk']] == sorted(r['tracks'])
    for tid, cls, first, cnt, dyn, off in g['trk']:
        t = r['tracks'][int(tid)]
        sl = slice(off, off + cnt)
        assert np.array_equal(t['frame'], g['ent_frame'][sl]) and np.array_equal(t['hit'], g['ent_hit'][sl]), tid
        assert (t['cls'] == cls).all() and (t['state'] == 'dynamic') == bool(dyn), tid
        assert np.abs(t['boxes_global'] - g['ent_box'][sl]).max() < 1e-5, tid
        assert np.abs(t['score'] - g['ent_score'][sl]).max() < 1e-5, tid
    # what the scene is there to exercise
    assert set(g['ent_hit']) == {0, 1, 2} and 0 < g['trk'][:, 4].sum() < len(g['trk'])
    assert g['counts'][25] == 0


def _two_frames(shift):
    """a vehicle detected twice, the second time `shift` metres further along its heading"""
    poses = np.tile(np.eye(4), (2, 1, 1))
    poses[:, :3, 3] = [5000.0, -3000.0, 50.0]
    boxes = np.zeros((2, 4, 9), np.float32)
    boxes[0, 0] = [10.0, 5.0, -1.0, 4.0, 2.0, 1.6, 0.0, 0.8, 1]
    boxes[1, 0] = [10.0 + shift, 5.0, -1.0, 4.0, 2.0, 1.6, 0.0, 0.8, 1]
    return boxes, np.array([1, 1], np.int32), poses


def test_margin_reports_a_decision_on_its_threshold():
    s = 3.2 / 1.2                                  # (4 - s) / (4 + s) = 0.2: the IoU sits on FIRST_STAGE.DIST_THRESHOLD
    r = track_ref.track_sequence(*_two_frames(s), tracker_cfg())
    assert r['margin'].value < 1e-3 and r['margin'].where == 'stage 1 iou', (r['margin'].value, r['margin'].where)
    r = track_ref.track_sequence(*_two_frames(1.0), tracker_cfg())
    assert r['margin'].value > 1e-2


def test_leading_empty_frames_are_empty():
    # the reference's reverse pass raises KeyError here; the oracle (and the device) give these frames no entries
    d = synthetic.synthetic_detections(7, frames=20, objects=30, false_positives=5)
    d['counts'][:3] = 0
    r = track_ref.track_sequence(d['boxes'], d['counts'], d['poses'], tracker_cfg())
    assert r['tracks'] and min(int(t['frame'][0]) for t in r['tracks'].values()) >= 3

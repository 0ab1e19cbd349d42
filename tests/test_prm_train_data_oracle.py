"""Host restatement of the PRM training samples (tests/prm_train_data_ref.py) against the reference's own training-branch
WaymoPositionDataset.extract_track_feature fed the same draws (tests/golden/prm_train_data.npz, written by
tests/golden/make_golden_prm_train_data.py); the statistics of the PRM's keyed draws; and refine.data.training_order('prm')."""
import os

import numpy as np
import pytest
import torch
from scipy import stats

from detzero_b200.refine import data as D
from oracle import refine_data_ref as R
from oracle import refine_train_data_ref as T
from tests import prm_train_data_ref as PT

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'prm_train_data.npz')
P_MIN = 1e-3            # every chi-square test: both tails above this


def _tracks():
    g = np.load(GOLD)
    pts, off = g['points'], g['frame_offsets']
    frames = np.zeros((len(pts), 6), np.float32)
    frames[:, 0] = np.repeat(np.arange(len(off) - 1), np.diff(off))
    frames[:, 1:5] = pts
    seed, epoch = int(g['seed']), int(g['epoch'])
    for b, L in enumerate(g['box_num']):
        L = int(L)
        crops = R.track_crops(frames, off, g['poses'], g['boxes'][b], g['frame_of_box'][b], L)
        yield g, b, L, PT.position_train_track(crops, g['boxes'][b], g['scores'][b], g['gt_boxes'][b], g['matched'][b], L,
                                               int(g['track_uid'][b]), seed, epoch)


def _close(a, b, tol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max() if a.size else 0.0
    assert err <= tol, err


def test_golden_covers_the_cases():
    seen = set()
    for g, b, L, r in _tracks():
        m = int(g['matched'][b, :L].sum())
        n = r['box_num']
        if m < 5:
            assert n == m
            seen.add('all kept')
        if L == 1:
            seen.add('one box')
        if m < L:
            seen.add('unmatched slots')
        if r['init_slot'] != n // 2:
            seen.add('init off centre')
        if n < m:
            seen.add('subset')
    assert seen == {'all kept', 'one box', 'unmatched slots', 'init off centre', 'subset'}, seen


def test_draws_match_golden():
    for g, b, L, r in _tracks():
        assert np.array_equal(r['kept'], g['prm_kept_%d' % b])
        assert r['init_slot'] == int(g['prm_init_%d' % b])
        assert r['box_num'] == int(g['prm_box_num_%d' % b])


def test_position_features_match_reference():
    for g, b, L, r in _tracks():
        rows = g['prm_rows_%d' % b]
        _close(r['pos_query_points'][rows], g['prm_pos_query_points_%d' % b])
        _close(r['pos_memory_points'][rows], g['prm_pos_memory_points_%d' % b])
        for k in ('pos_trajectory', 'gt_pos_trajectory', 'pos_init_box'):
            _close(r[k], g['prm_%s_%d' % (k, b)])
        assert np.array_equal(r['padding_mask'].astype(np.float32), g['prm_padding_mask_%d' % b])


def _chi2_ok(counts, expected, var=None):
    counts, expected = np.asarray(counts, np.float64), np.asarray(expected, np.float64)
    chi2 = ((counts - expected) ** 2 / (expected if var is None else var)).sum()
    dof = len(counts) - 1
    assert stats.chi2.sf(chi2, dof) > P_MIN and stats.chi2.cdf(chi2, dof) > P_MIN, (chi2, dof)


DRAWS = 12000


@pytest.fixture(scope='module')
def draws():
    """one PRM draw per (seed, epoch, uid) over many keys, through position_train_track itself: m = 13 matched of 20 slots"""
    L = 20
    matched = np.zeros(L, np.uint8)
    elig = np.array([0, 1, 3, 4, 6, 7, 9, 11, 12, 14, 15, 17, 19])
    matched[elig] = 1
    boxes = np.zeros((L, 7))
    boxes[:, 0], boxes[:, 3:6] = np.arange(L), 1.0
    crops = [np.zeros((0, 4))] * L
    out = []
    for d in range(DRAWS):
        seed, epoch, uid = d % 7, d // 7, 1000 + d % 5
        out.append(PT.position_train_track(crops, boxes, np.ones(L), boxes, matched, L, uid, seed, epoch, Lmax=L, kq=1, km=1))
    return elig, out


def test_kept_count_uniform(draws):
    elig, out = draws
    m = len(elig)
    n = np.array([o['box_num'] for o in out])
    assert n.min() >= 5 and n.max() <= m
    _chi2_ok(np.bincount(n - 5, minlength=m - 4), np.full(m - 4, DRAWS / (m - 4)))


def test_kept_slots_matched_uniform_and_sorted(draws):
    elig, out = draws
    hits = np.zeros(20)
    for o in out:
        k = o['kept']
        assert np.all(np.diff(k) > 0) and np.isin(k, elig).all()
        hits[k] += 1
    p = np.array([o['box_num'] for o in out]) / len(elig)
    _chi2_ok(hits[elig], np.full(len(elig), p.sum()), np.full(len(elig), (p * (1 - p)).sum()))


def test_init_position_uniform(draws):
    """the init box is a kept position, uniform over the kept count: binned on [0, 1) in 10 bins, each bin's mass known per n; and
    it is the box the trajectory's frame is centred on"""
    _, out = draws
    exp = np.zeros(10)
    at = []
    for o in out:
        n = o['box_num']
        assert 0 <= o['init_slot'] < n
        assert np.allclose(o['pos_trajectory'][o['init_slot'], [0, 1, 2, 6]], 0)
        exp += np.bincount((np.arange(n) * 10) // n, minlength=10) / n
        at.append(o['init_slot'] / n)
    _chi2_ok(np.bincount((np.array(at) * 10 + 1e-9).astype(int), minlength=10), exp)


def test_draw_is_the_crm_rule_on_the_matched_slots():
    """the PRM draw is train_draw's CRM rule with the matched slots as the eligible set, keyed on (seed, epoch, track_uid) only"""
    L = 40
    matched = (np.arange(L) % 3 != 1).astype(np.uint8)
    boxes = np.zeros((L, 7))
    boxes[:, 3:6] = 1.0
    crops = [np.zeros((0, 4))] * L
    for seed, epoch, uid in ((5, 0, 77), (5, 1, 77), (6, 0, 77), (5, 0, 78)):
        r = PT.position_train_track(crops, boxes, np.ones(L), boxes, matched, L, uid, seed, epoch, Lmax=L, kq=1, km=1)
        d = T.train_draw('crm', np.nonzero(matched)[0], uid, seed, epoch)
        assert np.array_equal(r['kept'], d['kept']) and r['init_slot'] == d['init']


def test_ground_truth_in_the_init_frame():
    """gt_pos_trajectory: the kept ground truth through init_coords_transform, heading limited before and after, at headings that
    cross +-pi"""
    L = 6
    boxes = np.zeros((L, 7))
    boxes[:, 0], boxes[:, 3:6] = np.arange(L) * 2.0, [4.0, 2.0, 1.5]
    boxes[:, 6] = [3.1, -3.1, 3.0, 0.0, -3.14, 7.0]
    gt = boxes.copy()
    gt[:, 1] += 0.3
    gt[:, 6] = [-3.1, 3.1, 9.0, -7.0, 3.14, 0.5]
    r = PT.position_train_track([np.zeros((0, 4))] * L, boxes, np.ones(L), gt, np.ones(L), L, 3, 1, 2, Lmax=8, kq=1, km=1)
    n, at, kept = r['box_num'], r['init_slot'], r['kept']
    yi = R.limit_heading(boxes[kept[at], 6])
    assert np.isclose(r['pos_init_box'][6], yi)
    for i, j in enumerate(kept):
        d = gt[j, :2] - boxes[kept[at], :2]
        c, s = np.cos(yi), np.sin(yi)
        assert np.allclose(r['gt_pos_trajectory'][i, :2], [c * d[0] + s * d[1], -s * d[0] + c * d[1]])
        h = r['gt_pos_trajectory'][i, 6]
        assert -np.pi <= h < np.pi and np.isclose(np.cos(h), np.cos(gt[j, 6] - yi)) and np.isclose(np.sin(h), np.sin(gt[j, 6] - yi))
    assert not r['gt_pos_trajectory'][n:].any() and not r['pos_trajectory'][n:].any()


class _Targets:
    def __init__(self, matched, matched_tracklet):
        self.matched = torch.as_tensor(matched, dtype=torch.uint8)
        self.matched_tracklet = torch.as_tensor(matched_tracklet, dtype=torch.uint8)


def test_training_order_prm_composition():
    g = np.random.default_rng(4)
    B, L = 40, 12
    mt = g.random(B) < 0.6
    matched = (g.random((B, L)) < 0.7) & mt[:, None]
    matched[np.nonzero(mt)[0][:3]] = False                      # matched tracklets with no matched box
    t = _Targets(matched, mt)
    o = D.training_order(t, 'prm', seed=3, epoch=2)
    want = np.nonzero(mt & matched.any(1))[0]
    assert sorted(o.tolist()) == want.tolist() and len(want) < mt.sum()
    assert np.array_equal(o, D.training_order(t, 'grm', seed=3, epoch=2))
    assert np.array_equal(o, D.training_order(t, 'prm', seed=3, epoch=2))
    assert not np.array_equal(o, D.training_order(t, 'prm', seed=3, epoch=3))
    with pytest.raises(ValueError, match="'prm'"):
        D.training_order(t, 'position', seed=3, epoch=2)

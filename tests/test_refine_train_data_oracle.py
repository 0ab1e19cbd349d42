"""Host restatement of the refiner training samples (oracle/refine_train_data_ref.py train_draw, geometry_train_track,
confidence_train_track) against the reference's own training-branch extract_track_feature fed the same draws
(tests/golden/refine_train_data.npz, written by tests/golden/make_golden_refine_train_data.py); the statistics of the keyed draws;
and the composition of refine.data.training_order."""
import os

import numpy as np
import pytest
import torch
from scipy import stats

from detzero_b200.refine import data as D
from oracle import refine_data_ref as R
from oracle import refine_train_data_ref as T

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'refine_train_data.npz')
MEM_STRIDE = 8          # the golden keeps every 8th GRM memory row
P_MIN = 1e-3            # every chi-square test: both tails above this


def _frames(g):
    pts, off = g['points'], g['frame_offsets']
    f = np.zeros((len(pts), 6), np.float32)
    f[:, 0] = np.repeat(np.arange(len(off) - 1), np.diff(off))
    f[:, 1:5] = pts
    return f


def _tracks():
    g = np.load(GOLD)
    frames = _frames(g)
    seed, epoch = int(g['seed']), int(g['epoch'])
    for b, L in enumerate(g['box_num']):
        L = int(L)
        crops = R.track_crops(frames, g['frame_offsets'], g['poses'], g['boxes'][b], g['frame_of_box'][b], L)
        grm = T.geometry_train_track(crops, g['boxes'][b], g['scores'][b], g['gt_boxes'][b], g['matched'][b], L,
                                     int(g['track_uid'][b]), seed, epoch)
        crm = T.confidence_train_track(crops, g['boxes'][b], g['scores'][b], g['iou'][b], L, int(g['track_uid'][b]), seed, epoch)
        yield g, b, L, grm, crm


def _close(a, b, tol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max() if a.size else 0.0
    assert err <= tol, err


def test_golden_covers_the_cases():
    seen = set()
    for g, b, L, grm, crm in _tracks():
        m = int(g['matched'][b, :L].sum())
        if m < 5:
            assert len(grm['kept']) == m and len(crm['kept']) == L
            seen.add('all kept')
        if L == 1:
            assert grm['geo_query_num'] == 1
            seen.add('one box')
        if m < L:
            seen.add('unmatched slots')
        if grm['flip'].any() and not grm['flip'].all():
            seen.add('flipped and unflipped')
        if crm['init_slot'] != len(crm['kept']) // 2:
            seen.add('init off centre')
    assert seen == {'all kept', 'one box', 'unmatched slots', 'flipped and unflipped', 'init off centre'}, seen
    g = np.load(GOLD)
    iou = g['iou'][g['matched'] != 0]
    assert (iou < 0.25).any() and ((iou >= 0.25) & (iou < 0.5)).any() and (iou >= 0.5).any()


def test_draws_match_golden():
    for g, b, L, grm, crm in _tracks():
        assert np.array_equal(grm['kept'], g['grm_kept_%d' % b])
        assert np.array_equal(grm['query_slots'], g['grm_query_%d' % b])
        assert np.array_equal(grm['flip'], g['grm_flip_%d' % b])
        assert np.array_equal(crm['kept'], g['crm_kept_%d' % b])
        assert crm['init_slot'] == int(g['crm_init_%d' % b])


def test_geometry_features_match_reference():
    for g, b, L, grm, crm in _tracks():
        assert grm['geo_query_num'] == int(g['grm_geo_query_num_%d' % b])
        for k in ('geo_query_points', 'geo_query_boxes', 'gt_geo_query_boxes', 'geo_trajectory', 'gt_geo_trajectory'):
            _close(grm[k], g['grm_%s_%d' % (k, b)])
        _close(grm['geo_memory_points'][::MEM_STRIDE], g['grm_geo_memory_points_%d' % b])


def test_confidence_features_match_reference():
    for g, b, L, grm, crm in _tracks():
        rows = g['crm_rows_%d' % b]
        _close(crm['conf_points'][rows], g['crm_conf_points_%d' % b])
        assert np.array_equal(crm['conf_score'].astype(np.float32), g['crm_conf_score_%d' % b])
        assert np.array_equal(crm['iou'].astype(np.float32), g['crm_iou_%d' % b])
        assert crm['box_num'] == int(g['crm_box_num_%d' % b])


def _chi2_ok(counts, expected, var=None):
    """Pearson's statistic against chi-square with len - 1 dof; var: each count's variance where it is not its expectation (a slot
    of a draw without replacement is in with probability p, variance p (1 - p), not p)"""
    counts, expected = np.asarray(counts, np.float64), np.asarray(expected, np.float64)
    chi2 = ((counts - expected) ** 2 / (expected if var is None else var)).sum()
    dof = len(counts) - 1
    assert stats.chi2.sf(chi2, dof) > P_MIN and stats.chi2.cdf(chi2, dof) > P_MIN, (chi2, dof)


DRAWS = 12000


@pytest.fixture(scope='module')
def draws():
    """one GRM and one CRM draw per (seed, epoch, uid) over many keys: m = 13 eligible of 20 slots, L = 20"""
    elig = np.array([0, 1, 3, 4, 6, 7, 9, 11, 12, 14, 15, 17, 19])
    out = []
    for d in range(DRAWS):
        seed, epoch, uid = d % 7, d // 7, 1000 + d % 5
        out.append((T.train_draw('grm', elig, uid, seed, epoch), T.train_draw('crm', np.arange(20), uid, seed, epoch)))
    return elig, out


def test_kept_count_uniform(draws):
    elig, out = draws
    for i, m in ((0, len(elig)), (1, 20)):
        n = np.array([len(o[i]['kept']) for o in out])
        assert n.min() >= 5 and n.max() <= m
        _chi2_ok(np.bincount(n - 5, minlength=m - 4), np.full(m - 4, DRAWS / (m - 4)))


def test_kept_slots_uniform_and_sorted(draws):
    elig, out = draws
    hits = np.zeros(20)
    for g, _ in out:
        k = g['kept']
        assert np.all(np.diff(k) > 0) and np.isin(k, elig).all()
        hits[k] += 1
    # given n, each of the m eligible slots is kept with probability n / m
    assert hits[np.setdiff1d(np.arange(20), elig)].sum() == 0
    p = np.array([len(g['kept']) for g, _ in out]) / len(elig)
    _chi2_ok(hits[elig], np.full(len(elig), p.sum()), np.full(len(elig), (p * (1 - p)).sum()))


def test_query_and_init_uniform(draws):
    _, out = draws
    q = np.zeros(5)                 # the GRM queries among the first 5 kept positions (every draw keeps >= 5)
    qn = qv = 0
    init = []
    for g, c in out:
        n = len(g['kept'])
        assert len(g['query']) == 3 and len(np.unique(g['query'])) == 3 and np.all(np.diff(g['query']) > 0) and g['query'].max() < n
        for j in g['query']:
            if j < 5:
                q[j] += 1
        qn += 3 / n
        qv += 3 / n * (1 - 3 / n)
        init.append(c['init'] / len(c['kept']))
    _chi2_ok(q, np.full(5, qn), np.full(5, qv))
    # init position over its kept count: discrete uniform, binned on [0, 1) in 10 bins; n = 5..20 so each bin's mass is known
    exp = np.zeros(10)
    for g, c in out:
        n = len(c['kept'])
        exp += np.bincount((np.arange(n) * 10) // n, minlength=10) / n
    _chi2_ok(np.bincount((np.array(init) * 10 + 1e-9).astype(int), minlength=10), exp)


def test_flip_rate_half(draws):
    _, out = draws
    f = np.concatenate([g['flip'] for g, _ in out])
    _chi2_ok([int((f == 0).sum()), int((f == 1).sum())], [len(f) / 2, len(f) / 2])


def test_draw_keys():
    elig = np.arange(40)
    a = T.train_draw('grm', elig, 77, 5, 0)
    assert all(np.array_equal(a[k], T.train_draw('grm', elig, 77, 5, 0)[k]) for k in ('kept', 'query', 'flip'))
    diff = 0
    for e in range(1, 20):
        b = T.train_draw('grm', elig, 77, 5, e)
        diff += not np.array_equal(a['kept'], b['kept'])
    assert diff == 19
    assert T.epoch_seed(5, 1) != T.epoch_seed(5, 0) != T.epoch_seed(6, 0)
    assert D.epoch_seed(5, 3) == T.epoch_seed(5, 3)
    assert not np.array_equal(T.train_draw('grm', elig, 78, 5, 0)['kept'], a['kept'])


class _Targets:
    def __init__(self, matched, matched_tracklet):
        self.matched = torch.as_tensor(matched, dtype=torch.uint8)
        self.matched_tracklet = torch.as_tensor(matched_tracklet, dtype=torch.uint8)


def test_training_order_composition():
    g = np.random.default_rng(4)
    B, L = 40, 12
    mt = g.random(B) < 0.6
    matched = (g.random((B, L)) < 0.7) & mt[:, None]
    matched[np.nonzero(mt)[0][:3]] = False                      # matched tracklets with no matched box
    t = _Targets(matched, mt)
    o = D.training_order(t, 'grm', seed=3, epoch=2)
    want = np.nonzero(mt & matched.any(1))[0]
    assert sorted(o.tolist()) == want.tolist() and len(want) < mt.sum()
    assert np.array_equal(o, D.training_order(t, 'grm', seed=3, epoch=2))
    assert not np.array_equal(o, D.training_order(t, 'grm', seed=3, epoch=3))
    o = D.training_order(t, 'crm', seed=3, epoch=2)
    pos, neg = set(np.nonzero(mt)[0].tolist()), set(np.nonzero(~mt)[0].tolist())
    assert len(o) == 2 * len(pos)
    assert sorted(i for i in o.tolist() if i in pos) == sorted(pos)
    assert sum(i in neg for i in o.tolist()) == len(pos)
    with pytest.raises(ValueError, match='negative'):
        D.training_order(_Targets(matched, np.ones(B, bool)), 'crm', seed=3, epoch=2)


def test_training_order_negatives_uniform():
    B = 10
    mt = np.zeros(B, bool)
    mt[:4] = True
    t = _Targets(np.zeros((B, 3), bool), mt)
    hits = np.zeros(B)
    for e in range(2000):
        o = D.training_order(t, 'crm', seed=1, epoch=e)
        for i in o:
            if not mt[i]:
                hits[i] += 1
    _chi2_ok(hits[4:], np.full(6, 2000 * 4 / 6))

"""Host restatement of the refiner input builder (oracle/refine_data_ref.py) against the reference's own extract_track_feature /
revert_to_each_frame outputs (tests/golden/refine_data.npz, written by tests/golden/make_golden_refine_data.py), and the keyed
sampler's properties."""
import os

import numpy as np
from scipy import stats

from oracle import refine_data_ref as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'refine_data.npz')


MEM_STRIDE = 8          # the golden keeps every 8th GRM memory row


def _frames(g):
    """collated rows [frame, x, y, z, tanh(i), 0] from the stored [x, y, z, tanh(i)] points and frame offsets"""
    pts, off = g['points'], g['frame_offsets']
    f = np.zeros((len(pts), 6), np.float32)
    f[:, 0] = np.repeat(np.arange(len(off) - 1), np.diff(off))
    f[:, 1:5] = pts
    return f


def _tracks():
    g = np.load(GOLD)
    frames = _frames(g)
    for b, L in enumerate(g['box_num']):
        L = int(L)
        crops = R.track_crops(frames, g['frame_offsets'], g['poses'], g['boxes'][b], g['frame_of_box'][b], L)
        yield g, b, L, crops


def test_golden_covers_the_cases():
    g = np.load(GOLD)
    assert sorted(int(v) for v in g['box_num']) == [1, 2, 9, 200]
    counts = np.concatenate([g['counts_%d' % b] for b in range(len(g['box_num']))])
    for lo, hi in ((0, 1), (1, 48), (48, 256), (256, 2049), (2049, 1 << 30)):
        assert ((counts >= lo) & (counts < hi)).any(), (lo, hi)
    h = g['boxes'][0, :200, 6]
    assert h.max() > np.pi and h.min() < np.pi                 # headings cross +-pi
    assert 3 in g['cls']


def test_crop_counts_and_selections_match_golden():
    for g, b, L, crops in _tracks():
        assert np.array_equal([len(c) for c in crops], g['counts_%d' % b])
        uid, seed = int(g['track_uid'][b]), int(g['seed'])
        o = R.position_track(crops, g['boxes'][b], g['scores'][b], L, g['cls'][b], uid, seed)
        assert np.array_equal(np.concatenate(o['sel'][0]), g['prm_sel_q_%d' % b])
        assert np.array_equal(np.concatenate(o['sel'][1]), g['prm_sel_m_%d' % b])
        o = R.confidence_track(crops, g['boxes'][b], g['scores'][b], L, uid, seed)
        assert np.array_equal(np.concatenate(o['sel']), g['crm_sel_%d' % b])
        o = R.geometry_track(crops, g['boxes'][b], g['scores'][b], L, uid, seed)
        assert np.array_equal(np.concatenate(o['sel'][0]), g['grm_sel_q_%d' % b])
        assert np.array_equal(o['sel'][1], g['grm_sel_m_%d' % b])


def _close(a, b, tol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    err = np.abs(a - b).max() if a.size else 0.0
    assert err <= tol, err


def test_features_match_reference():
    for g, b, L, crops in _tracks():
        uid, seed, keep = int(g['track_uid'][b]), int(g['seed']), g['keep_%d' % b]
        bx, sc = g['boxes'][b], g['scores'][b]
        o = R.position_track(crops, bx, sc, L, g['cls'][b], uid, seed)
        _close(o['pos_query_points'][keep], g['prm_pos_query_points_%d' % b])
        _close(o['pos_memory_points'][keep], g['prm_pos_memory_points_%d' % b])
        _close(o['pos_trajectory'], g['prm_pos_trajectory_%d' % b])
        assert np.array_equal(o['padding_mask'], g['prm_padding_mask_%d' % b])
        _close(o['pos_init_box'], g['prm_pos_init_box_%d' % b])
        if int(g['cls'][b]) == 3:
            o = R.position_track(crops, bx, sc, L, g['cls'][b], uid, seed, with_class=True)
            _close(o['pos_query_points'][keep], g['prmc_pos_query_points_%d' % b])
            _close(o['pos_memory_points'][keep], g['prmc_pos_memory_points_%d' % b])
        o = R.confidence_track(crops, bx, sc, L, uid, seed)
        _close(o['conf_points'][keep], g['crm_conf_points_%d' % b])
        assert np.array_equal(o['conf_score'].astype(np.float32), g['crm_conf_score_%d' % b])
        o = R.geometry_track(crops, bx, sc, L, uid, seed)
        assert o['geo_query_num'] == int(g['grm_geo_query_num_%d' % b])
        _close(o['geo_query_points'], g['grm_geo_query_points_%d' % b])
        _close(o['geo_query_boxes'], g['grm_geo_query_boxes_%d' % b])
        _close(o['geo_memory_points'][::MEM_STRIDE], g['grm_geo_memory_points_%d' % b])


def test_revert_matches_reference():
    for g, b, L, crops in _tracks():
        poses = g['poses'][g['frame_of_box'][b, :L]]
        lid, wor = R.revert_position(g['prm_pred_%d' % b], g['boxes'][b], L, poses)
        _close(wor, g['prm_revert_world_%d' % b])
        _close(lid, g['prm_revert_lidar_%d' % b])
        lid, _ = R.revert_geometry(g['grm_pred_%d' % b], g['boxes'][b], L, poses)
        _close(lid, g['grm_revert_lidar_%d' % b])


def test_sampler_ranks():
    for n, k in ((1000, 256), (257, 256), (5000, 48), (10 ** 6, 4096)):
        r = R.sample_ranks(n, k, 5, 123456789, 7, R.PRM_Q)
        assert len(r) == k and len(np.unique(r)) == k and np.all(np.diff(r) > 0) and r.min() >= 0 and r.max() < n
        assert np.array_equal(r, R.sample_ranks(n, k, 5, 123456789, 7, R.PRM_Q))          # same key, same ranks
        assert not np.array_equal(r, R.sample_ranks(n, k, 5, 123456789, 7, R.PRM_M))
    for n in (0, 1, 47, 256):
        assert np.array_equal(R.sample_ranks(n, 256, 1, 2, 3, R.CRM_Q), np.arange(n))
    assert R.mix64_int(0) == 0xE220A8397B1DCDAF                                           # splitmix64's first output for state 0
    assert int(R.mix64(np.uint64(12345))) == R.mix64_int(12345)
    assert len(np.unique(R.mix64(np.arange(1 << 16, dtype=np.uint64)))) == 1 << 16


def test_sampler_inclusion_is_uniform():
    n, k, draws = 1000, 256, 20000
    hits = np.zeros(n)
    for d in range(draws):
        hits[R.sample_ranks(n, k, 11, d, d % 200, R.PRM_Q)] += 1
    expected = draws * k / n
    # each rank's count is Binomial(draws, k / n) with variance expected * (1 - k / n); the counts sum to draws * k (n - 1 dof)
    chi2 = ((hits - expected) ** 2 / (expected * (1 - k / n))).sum()
    assert stats.chi2.sf(chi2, n - 1) > 1e-3 and stats.chi2.cdf(chi2, n - 1) > 1e-3, chi2

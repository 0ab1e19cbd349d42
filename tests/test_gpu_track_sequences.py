"""detzero_b200.track.track_sequences (csrc/tracker.cu) against the numpy restatement of the DetZero tracker (oracle/track_ref.py).

Each scene is built so that the oracle's decision margin is at least 1e-3; the device must then take every decision the oracle takes:
the same track ids, entry frames, hit flags, classes, motion states and overlap-filter keep flags.  Boxes agree within 5e-3 m and
1e-4 rad (the KF state is float32 at km world offsets), scores exactly."""
import os

import numpy as np
import pytest
import torch

from detzero_b200 import synthetic
from detzero_b200.track import tracker_cfg, track_sequences
from oracle import track_ref

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'track.npz')


def _oracle(d):
    r = track_ref.track_sequence(d['boxes'], d['counts'], d['poses'], tracker_cfg())
    assert r['margin'].value >= 1e-3, (r['margin'].value, r['margin'].where)
    return r


def _run(ds, **kw):
    F = max(len(d['counts']) for d in ds)
    K = max(d['boxes'].shape[1] for d in ds)
    boxes = np.zeros((len(ds), F, K, 9), np.float32)
    counts = np.zeros((len(ds), F), np.int32)
    poses = np.tile(np.eye(4), (len(ds), F, 1, 1))
    for s, d in enumerate(ds):
        f = len(d['counts'])
        boxes[s, :f, :d['boxes'].shape[1]] = d['boxes']
        counts[s, :f], poses[s, :f] = d['counts'], d['poses']
    return track_sequences(torch.from_numpy(boxes).cuda(), torch.from_numpy(counts), torch.from_numpy(poses),
                           num_frames=[len(d['counts']) for d in ds], **kw)


def _compare(res, s, ref, d):
    track_ref.check_device(res, s, ref)


def test_device_vs_reference_golden():
    g = np.load(GOLDEN)
    ref = {'kept': [g['kept'][f, :c] for f, c in enumerate(g['counts'])], 'tracks': {}}
    for tid, cls, first, cnt, dyn, off in g['trk']:
        sl = slice(off, off + cnt)
        ref['tracks'][int(tid)] = {'frame': g['ent_frame'][sl], 'hit': g['ent_hit'][sl], 'cls': np.full(cnt, cls),
                                   'state': 'dynamic' if dyn else 'static', 'boxes_global': g['ent_box'][sl],
                                   'score': g['ent_score'][sl]}
    d = {'boxes': g['boxes'], 'counts': g['counts'], 'poses': g['poses']}
    _compare(_run([d]), 0, ref, d)


@pytest.mark.parametrize('seed', [1, 2, 4])
def test_small_scene_vs_oracle(seed):
    d = synthetic.synthetic_detections(seed, frames=30, objects=40, false_positives=10, chain=6)
    ref = _oracle(d)
    _compare(_run([d]), 0, ref, d)


def test_full_scale_vs_oracle_batched():
    ds = [synthetic.synthetic_detections(seed, frames=199, objects=300, false_positives=40) for seed in (11, 15)]
    res = _run(ds)
    for s, d in enumerate(ds):
        _compare(res, s, _oracle(d), d)


def test_alone_equals_batched_and_runs_are_bit_equal():
    ds = [synthetic.synthetic_detections(seed, frames=40, objects=60, false_positives=20, chain=5) for seed in (21, 22, 23)]
    a, b = _run(ds), _run(ds)
    alone = _run([ds[1]])
    for t in ('trk', 'ent_box', 'ent_score', 'ent_hit', 'ent_frame', 'kept'):
        assert torch.equal(getattr(a, t), getattr(b, t)), t
        assert torch.equal(getattr(a, t)[1], getattr(alone, t)[0]), t


def test_edge_cases():
    # F = 1: every kept detection births a track; none survives LEAST_AGE
    d = synthetic.synthetic_detections(3, frames=1, objects=20, false_positives=5)
    res = _run([d])
    assert res.tracks(0).shape[0] == 0
    # a full K = 500 frame, empty frames after the first, an all-low-score sequence
    d = synthetic.synthetic_detections(5, frames=20, objects=60, false_positives=470)
    assert d['counts'].max() == 500
    d['counts'][[4, 9]] = 0
    _compare(_run([d]), 0, _oracle(d), d)
    low = synthetic.synthetic_detections(6, frames=20, objects=30, false_positives=5)
    low['boxes'][..., 7] = np.minimum(low['boxes'][..., 7], 0.05)
    _compare(_run([low]), 0, _oracle(low), low)


def test_leading_empty_frames():
    d = synthetic.synthetic_detections(7, frames=20, objects=30, false_positives=5)
    d['counts'][:3] = 0
    ref = _oracle(d)
    _compare(_run([d]), 0, ref, d)
    assert min(t['frame'][0] for t in ref['tracks'].values()) >= 3


def test_capacity_overflow_raises():
    d = synthetic.synthetic_detections(8, frames=10, objects=40, false_positives=5)
    with pytest.raises(RuntimeError, match='max_tracks'):
        _run([d], max_tracks=16)
    with pytest.raises(RuntimeError, match='max_entries'):
        _run([d], max_entries=64)


def _chain_scene(n=300, gap=20, frames=8):
    """n + 1 static pedestrians 0.73 m apart in a line: every detection overlaps three tracks (IoU 0.104 with each neighbour, over
    the 0.1 threshold), so a frame is one component of n rows and n columns.  Frame 0 has members 0..n-1; every later frame misses
    member `gap` and has member n.  Keeping n matches then takes an augmenting path: the detections gap+1..n each move one track
    down the chain."""
    d = synthetic.synthetic_detections(31, frames=frames, objects=0, false_positives=0, chain=n + 1)
    for f in range(frames):
        c = d['counts'][f]
        keep = d['gt_id'][f, :c] != (n if f == 0 else gap)
        rows = d['boxes'][f, :c][keep]
        d['boxes'][f] = 0
        d['boxes'][f, :len(rows)] = rows
        d['counts'][f] = len(rows)
    return d


def test_large_component_vs_scipy():
    # the oracle assigns with scipy.optimize.linear_sum_assignment on the reference's 1 - IoU / 5000 costs; the device solves the
    # 300 x 300 component block-wide
    d = _chain_scene()
    ref = _oracle(d)
    assert len(ref['tracks']) == 300                                     # member n never births a track: it takes one
    last = ref['tracks'][299]
    assert abs(last['boxes_global'][1, 0] - last['boxes_global'][0, 0] - 0.73) < 1e-3
    _compare(_run([d]), 0, ref, d)


def _detections_from_sequence(s, seed, miss=0.1, fp=10, K=500):
    """lidar detections of a synthetic_sequence's ground-truth boxes: 3 cm / 0.01 rad jitter, about `miss` of the boxes missed
    (never the first or last two of a track), `fp` far false positives per frame, rows shuffled.  -> boxes, counts, gt (F, K)"""
    g = np.random.default_rng([seed, 0xE2E])
    F = len(s['poses'])
    dims = [[4.7, 2.0, 1.6], [0.9, 0.9, 1.8], [1.9, 0.8, 1.7]]
    rows = [[] for _ in range(F)]
    for b in range(len(s['box_num'])):
        n = int(s['box_num'][b])
        for j in range(n):
            if 2 <= j < n - 2 and g.random() < miss:
                continue
            f = int(s['frame_of_box'][b, j])
            P, w = s['poses'][f], s['boxes'][b, j]
            loc = (w[:3] + g.normal(0, 0.03, 3) - P[:3, 3]) @ P[:3, :3]
            h = w[6] + g.normal(0, 0.01) - np.arctan2(P[1, 0], P[0, 0])
            rows[f].append(([*loc, *(w[3:6] * (1 + g.normal(0, 0.005, 3))), np.arctan2(np.sin(h), np.cos(h)),
                             g.uniform(0.3, 0.95), s['cls'][b]], b))
    for f in range(F):
        for _ in range(fp):
            a, r, c = g.uniform(-np.pi, np.pi), g.uniform(300, 500), int(g.integers(1, 4))
            rows[f].append(([r * np.cos(a), r * np.sin(a), -1.0, *dims[c - 1], g.uniform(-np.pi, np.pi), g.uniform(0.02, 0.3), c], -1))
    boxes, gt, counts = np.zeros((F, K, 9), np.float32), np.full((F, K), -1), np.zeros(F, np.int32)
    for f in range(F):
        for i, k in enumerate(g.permutation(len(rows[f]))):
            boxes[f, i], gt[f, i] = rows[f][k]
        counts[f] = len(rows[f])
    return boxes, counts, gt


@pytest.mark.parametrize('seed', [2, 4])
def test_end_to_end_ground_truth_to_prm(seed):
    """synthetic_sequence ground truth -> jittered, shuffled detections with misses and far false positives -> the tracker: every
    ground-truth track comes out as exactly one track over exactly its frames, whose updated boxes are its detections; then
    .track_batch() -> position_inputs on the sequence's points -> PRM forward"""
    from detzero_b200.refine import PositionTransformer
    from detzero_b200.refine import data as rdata
    from oracle import weights
    F = 40
    lengths = [int(x) for x in np.random.default_rng(seed).integers(8, F + 1, 12)]
    s = synthetic.synthetic_sequence(seed, frames=F, tracks=12, n_background=2000, ego_step=0.0, max_speed=0.3, lengths=lengths)
    boxes, counts, gt = _detections_from_sequence(s, seed)
    res = track_sequences(torch.from_numpy(boxes).cuda(), torch.from_numpy(counts), torch.from_numpy(s['poses']))
    eb, eh, ef = res.ent_box[0].cpu().numpy(), res.ent_hit[0].cpu().numpy(), res.ent_frame[0].cpu().numpy()
    owner = {}
    for tid, cls, first, cnt, dyn, off in res.tracks(0):
        for o in range(off, off + cnt):
            if eh[o] != 1:
                continue
            f = ef[o]
            live = [b for b in range(len(lengths)) if s['frame_of_box'][b, 0] <= f < s['frame_of_box'][b, 0] + s['box_num'][b]]
            dist = [np.linalg.norm(s['boxes'][b, f - s['frame_of_box'][b, 0], :2] - eb[o, :2]) for b in live]
            assert live and min(dist) < 0.3, (tid, f)
            b = live[int(np.argmin(dist))]
            assert cls == s['cls'][b]
            owner.setdefault(b, set()).add(int(tid))
    rows = {int(r[0]): r for r in res.tracks(0)}
    assert len(rows) == len(lengths)
    for b in range(len(lengths)):
        assert len(owner.get(b, ())) == 1, (b, owner.get(b))
        tid = next(iter(owner[b]))
        _, _, first, cnt, _, off = rows[tid]
        assert np.array_equal(ef[off:off + cnt], s['frame_of_box'][b, :s['box_num'][b]]), b
    tb = res.track_batch(L=200)
    assert sorted(tb.box_num.cpu().tolist()) == sorted(lengths)
    cfg = synthetic.prm_cfg()
    cfg.COMPUTE_MODE = 'fp32'
    m = PositionTransformer(cfg, 32, 32).eval()
    weights.load_seeded(m, seed)
    m = m.cuda()
    inp = rdata.position_inputs(torch.from_numpy(s['frames']).cuda(), s['frame_offsets'], torch.from_numpy(s['poses']).cuda(), tb,
                                seed=seed)
    with torch.no_grad():
        pred = m(dict(inp))['batch_box_preds']
    assert pred.shape[:2] == (len(tb), 200)
    valid = inp['padding_mask'] == 0
    assert int(valid.sum()) == sum(lengths) and torch.isfinite(pred[valid]).all()


def test_to_reference_forms():
    d = synthetic.synthetic_detections(9, frames=30, objects=20, false_positives=5)
    res = _run([d])
    tracks, drops = res.to_reference(['seq'], [[str(f) for f in range(30)]])
    assert sorted(tracks['seq']) == [int(r[0]) for r in res.tracks(0)]
    for tid, cls, first, cnt, dyn, off in res.tracks(0):
        t = tracks['seq'][int(tid)]
        assert len(t['boxes_global']) == cnt and t['sample_idx'][0] == str(first) and (t['obj_ids'] == tid).all()
        assert t['state'] == ('dynamic' if dyn else 'static') and set(t['name']) == {('Vehicle', 'Pedestrian', 'Cyclist')[cls - 1]}
    n_drop = sum(int((~res.kept[0, f, :c]).sum()) for f, c in enumerate(d['counts']))
    assert sum(len(v['score']) for v in drops['seq'].values()) == n_drop
    tb = res.track_batch('Vehicle')
    assert sorted(int(r[0]) for r in res.tracks(0) if r[1] == 1) == sorted(tb.track_uid.cpu().tolist())

"""detzero_b200.track.assign_track_target / tracklet_recall (csrc/track_gt.cu) against the reference's golden vectors
(tests/golden/track_gt.npz) and the numpy restatement (oracle/track_gt_ref.py).

Where the oracle's decision margin is at least 1e-3 the device must take every decision it takes: the same matches, states, buckets
and recall table (integers exactly, and so the floats derived from them).  Per-entry IoUs agree within 1e-5 on the golden scene.  On
the synthetic ones, whose boxes lie up to 100 m from the sensor, the float32 polygon clip's corner coordinates carry ~1e-5 m ulps and
the device's sinf / cosf / atan2f are not the oracle's C library's; the clip counts a corner within 1e-2 m outside the other box as
inside, so an IoU jumps where a corner crosses that margin, and nearly coincident boxes make it ill-conditioned (the IoU can exceed
1).  There at most one entry in a thousand may differ by more than 5e-5, and none by 2e-2."""
import numpy as np
import pytest
import torch

from detzero_b200 import synthetic
from detzero_b200.track import (CLASS_NAMES, TrackResult, assign_track_target, ground_truth_from_infos, track_sequences,
                                tracklet_recall)
from oracle import track_gt_ref
from tests import track_gt_golden

pytestmark = pytest.mark.gpu
THR = {'Vehicle': 0.3, 'Pedestrian': 0.1, 'Cyclist': 0.1}


def _track_result(seqs, F):
    """a TrackResult of track dicts {id: {'boxes_global', 'name', 'sample_idx'}} (frame ids str(f)), one per sequence"""
    S = len(seqs)
    T = max([len(t) for t in seqs] + [1])
    E = max([sum(len(v['name']) for v in t.values()) for t in seqs] + [1])
    trk = np.zeros((S, T, 6), np.int32)
    eb, ef = np.zeros((S, E, 9)), np.zeros((S, E), np.int32)
    n = np.zeros(S, np.int32)
    for s, tracks in enumerate(seqs):
        off = 0
        for k, (tid, t) in enumerate(tracks.items()):
            c = len(t['name'])
            fr = [int(x) for x in t['sample_idx']]
            trk[s, k] = [tid, CLASS_NAMES.index(str(t['name'][0])) + 1, fr[0], c, 0, off]
            eb[s, off:off + c] = np.asarray(t['boxes_global'])[:, :9]
            ef[s, off:off + c] = fr
            off += c
        n[s] = len(tracks)
    d = lambda a: torch.from_numpy(a).cuda()
    return TrackResult(d(np.zeros((S, F, 1, 9), np.float32)), d(np.zeros((S, F), np.int32)), None, d(np.full(S, F, np.int32)),
                       d(trk), d(n), d(eb), d(np.full((S, E), 0.8, np.float32)), d(np.ones((S, E), np.int32)), d(ef),
                       d(np.zeros((S, F, 1), np.uint8)))


def _with_poses(tr, gt):
    tr.poses = gt.poses
    return tr


def _check_assign(res, names, scenes, min_margin=1e-3):
    out = res.to_reference(names)
    for name, (frames, tracks) in zip(names, scenes):
        ref, margin = track_gt_ref.assign_track_target(frames, tracks, THR)
        assert margin.value >= min_margin, (margin.value, margin.where)
        dev = out[name]
        assert list(dev['label']) == list(ref['label']) and list(dev['unlabel']) == list(ref['unlabel'])
        loose, total = 0, 0
        for tid, r in ref['label'].items():
            d = dev['label'][tid]
            assert d['track']['state'] == r['track']['state'], tid
            err = np.abs(d['track']['iou'] - r['track']['iou'])
            assert err.max() < 2e-2, (tid, err.max())
            loose += int((err > 5e-5).sum())
            total += len(err)
            for k in ('gt_boxes_global', 'gt_boxes_lidar', 'name', 'obj_ids', 'sample_idx'):
                assert np.array_equal(d['gt'][k], r['gt'][k]), (tid, k)
        assert loose <= max(1, total // 1000), (loose, total)


def _check_recall(table, scenes, min_margin=1e-3):
    ref, margin, _ = track_gt_ref.tracklet_recall(scenes)
    assert margin.value >= min_margin, (margin.value, margin.where)
    for d in ('l1', 'l2'):
        for c in CLASS_NAMES:
            for k in ('tp', 'fp', 'gt_nums', 'pred_nums', 'cutoffs', 'precisions', 'recalls'):
                assert list(table[d][c][k]) == list(ref[d][c][k]), (d, c, k)
    assert table['iou_thresholds'] == ref['iou_thresholds'] and table['method'] == '3d'


def test_device_vs_reference_golden():
    g, frames, tracks = track_gt_golden.load()
    gt = ground_truth_from_infos(frames, ['seq'])
    tr = _with_poses(_track_result([tracks], len(frames)), gt)
    out = assign_track_target(tr, gt).to_reference(['seq'])['seq']
    assert list(out['label']) == g['label_tk'].tolist() and list(out['unlabel']) == g['unlabel_tk'].tolist()
    assert [v['gt']['obj_ids'][0] for v in out['label'].values()] == g['label_obj'].tolist()
    assert [v['track']['state'] == 'dynamic' for v in out['label'].values()] == g['label_state'].tolist()
    assert np.abs(np.concatenate([v['track']['iou'] for v in out['label'].values()]) - g['label_iou']).max() < 1e-5
    assert np.array_equal(np.concatenate([v['gt']['sample_idx'] for v in out['label'].values()]), g['label_gt_sample_idx'])
    ref = track_gt_golden.recall_table(g)
    for table in (tracklet_recall(tr, gt), tracklet_recall({'seq': tracks}, gt)):
        for d in ('l1', 'l2'):
            for c in CLASS_NAMES:
                for k, v in ref[d][c].items():
                    assert np.array_equal(np.asarray(table[d][c][k]), v), (d, c, k)


def _scene(seed, frames=40, objects=30, S_bg=500, radius=45.0):
    s = synthetic.synthetic_sequence(seed, frames=frames, tracks=objects, n_background=S_bg, ego_step=0.5, max_speed=0.3,
                                     radius=radius)
    g = np.random.default_rng(seed)
    diff = [g.choice([0, 0, 0, 1, 2], 200) for _ in range(objects)]
    infos = synthetic.synthetic_ground_truth(s, seed, name='seq%d' % seed, difficulty=diff)
    boxes, counts, _ = synthetic.detections_from_sequence(s, seed)
    return s, infos, boxes, counts


def _tracked(scenes):
    F = max(len(sc[0]['poses']) for sc in scenes)
    boxes = np.zeros((len(scenes), F, 500, 9), np.float32)
    counts = np.zeros((len(scenes), F), np.int32)
    poses = np.tile(np.eye(4), (len(scenes), F, 1, 1))
    for i, (s, _, b, c) in enumerate(scenes):
        f = len(c)
        boxes[i, :f], counts[i, :f], poses[i, :f] = b, c, s['poses']
    return track_sequences(torch.from_numpy(boxes).cuda(), torch.from_numpy(counts), torch.from_numpy(poses),
                           num_frames=[len(sc[3]) for sc in scenes], max_entries=1 << 20)


def _run_and_check(seeds, min_margin=1e-3, **kw):
    scenes = [_scene(seed, **kw) for seed in seeds]
    names = ['seq%d' % seed for seed in seeds]
    res = _tracked(scenes)
    gt = ground_truth_from_infos([i for sc in scenes for i in sc[1]], names)
    tracks, _ = res.to_reference(names, gt.frame_ids)
    ref_scenes = [(sc[1], tracks[n]) for sc, n in zip(scenes, names)]
    _check_assign(assign_track_target(res, gt), names, ref_scenes, min_margin)
    _check_recall(tracklet_recall(res, gt), ref_scenes, min_margin)
    return res, gt


@pytest.mark.parametrize('seed', [1, 3])
def test_seeded_scene_vs_oracle(seed):
    _run_and_check([seed])


def test_full_scale_vs_oracle():
    # 300 objects over 199 frames give tens of thousands of IoUs, and the recall threshold 0.7 lies inside the spread of a jittered
    # detection's 3-D IoU with its own box, so no such scene keeps every IoU 1e-3 from its threshold.  This one keeps them 3e-4 away
    # (asserted at 1e-4), six times the bound on device-vs-oracle IoU differences.
    _run_and_check([5], min_margin=1e-4, frames=199, objects=300, S_bg=200, radius=100.0)


def test_alone_equals_batched_and_runs_are_bit_equal():
    scenes = [_scene(seed) for seed in (21, 22, 23)]
    names = ['seq21', 'seq22', 'seq23']
    res = _tracked(scenes)
    gt = ground_truth_from_infos([i for sc in scenes for i in sc[1]], names)
    a, b = assign_track_target(res, gt), assign_track_target(res, gt)
    res1 = _tracked(scenes[1:2])
    gt1 = ground_truth_from_infos(scenes[1][1], names[1:2])
    alone = assign_track_target(res1, gt1)
    for t in ('obj_rec', 'trk_rec', 'ent_iou'):
        assert torch.equal(getattr(a, t), getattr(b, t)), t
        x, y = getattr(a, t)[1], getattr(alone, t)[0]
        n = min(x.shape[0], y.shape[0])
        assert torch.equal(x[:n], y[:n]) and not x[n:].any() and not y[n:].any(), t
    assert tracklet_recall(res, gt) == tracklet_recall(res, gt)


def _chain(n=80, frames=4, seed=7):
    """n static pedestrians 0.6 m apart in a line and n tracks each 0.05..0.12 m beside one of them (a little further every
    frame): every inner track overlaps three objects above the 0.1 BEV threshold (IoU >= 0.106 with the farther neighbour), so the
    whole chain is one assignment component of about 3n edges"""
    g = np.random.default_rng(seed)
    pose = np.eye(4)
    pose[:3, 3] = [5000.0, -3000.0, 50.0]
    ids = ['p%03d' % i for i in range(n)]
    obj = np.array([[5000.0 + 0.6 * i, -3000.0, 49.0, 0.9, 0.9, 1.8, 0.0, 0.0, 0.0] for i in range(n)])
    infos = []
    for f in range(frames):
        lid = obj[:, :7].copy()
        lid[:, :3] -= pose[:3, 3]
        infos.append({'sequence_name': 'chain', 'sample_idx': f, 'pose': pose,
                      'annos': {'name': np.array(['Pedestrian'] * n), 'obj_ids': np.array(ids), 'gt_boxes_lidar': lid.astype(np.float32),
                                'gt_boxes_global': obj, 'difficulty': np.zeros(n, np.int32), 'num_points_in_gt': np.full(n, 50, np.int32)}})
    shift = g.uniform(0.05, 0.12, n)
    tracks = {}
    for k in range(n):
        b = np.repeat(obj[k:k + 1], frames, 0)
        b[:, 0] += shift[k] * (1 + 0.02 * np.arange(frames))
        tracks[k] = {'boxes_global': b, 'name': np.array(['Pedestrian'] * frames), 'sample_idx': np.array([str(f) for f in range(frames)])}
    return infos, tracks


def test_large_component_vs_scipy():
    infos, tracks = _chain()
    gt = ground_truth_from_infos(infos, ['chain'])
    tr = _with_poses(_track_result([tracks], len(infos)), gt)
    _check_assign(assign_track_target(tr, gt), ['chain'], [(infos, tracks)])
    res = assign_track_target(tr, gt)
    assert len(res.matches(0)) == 80


def test_capacity_overflow_raises():
    infos, tracks = _chain(n=20)
    gt = ground_truth_from_infos(infos, ['chain'])
    tr = _with_poses(_track_result([tracks], len(infos)), gt)
    with pytest.raises(RuntimeError, match='max_pairs'):
        assign_track_target(tr, gt, max_pairs=8)
    with pytest.raises(RuntimeError, match='max_pairs'):
        tracklet_recall(tr, gt, max_pairs=8)


def test_empty_sequences():
    infos, tracks = _chain(n=10)
    empty = [{'sequence_name': 'empty', 'sample_idx': f, 'pose': np.eye(4),
              'annos': {'name': np.array([], '<U10'), 'obj_ids': np.array([], '<U4'), 'gt_boxes_lidar': np.zeros((0, 7), np.float32),
                        'gt_boxes_global': np.zeros((0, 9)), 'difficulty': np.zeros(0, np.int32),
                        'num_points_in_gt': np.zeros(0, np.int32)}} for f in range(len(infos))]
    gt = ground_truth_from_infos(infos + empty, ['chain', 'empty'])
    tr = _with_poses(_track_result([tracks, {}], len(infos)), gt)
    out = assign_track_target(tr, gt).to_reference(['chain', 'empty'])
    assert out['empty'] == {'label': {}, 'unlabel': {}} and len(out['chain']['label']) == 10
    # ground truth but no tracks, tracks but no ground truth
    gt2 = ground_truth_from_infos(empty + infos, ['empty', 'chain'])
    tr2 = _with_poses(_track_result([tracks, {}], len(infos)), gt2)
    out = assign_track_target(tr2, gt2).to_reference(['empty', 'chain'])
    assert out['chain'] == {'label': {}, 'unlabel': {}} and len(out['empty']['unlabel']) == 10
    table = tracklet_recall(tr2, gt2)
    assert table['l1']['Pedestrian']['gt_nums'][0] == 10 and table['l1']['Pedestrian']['tp'] == [0] * 10
    assert table['l1']['Pedestrian']['pred_nums'][0] == 10

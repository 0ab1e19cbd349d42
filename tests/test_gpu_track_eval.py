"""detzero_b200.evaluate's tracking metrics (csrc/track_eval.cu) against the numpy restatement oracle/track_eval_ref.py: the int64
records (matches, misses, FP, mismatches exactly; the cost within the device-vs-oracle IoU bound of test_gpu_track_gt.py per
match) on seeded multi-sequence scenes whose every decision the oracle takes at least 1e-5 from its threshold, on the hand cases,
on one large assignment component; records do not depend on the run or on the grouping of sequences; the raw tracker output and
the offboard chain scored on the device equal the reference-shaped entry point on the same frames."""
import numpy as np
import pytest
import torch

from detzero_b200 import evaluate, offboard, synthetic
from detzero_b200.track import CLASS_NAMES, ground_truth_from_infos, track_sequences
from oracle import track_eval_ref, track_gt_ref
from tests import track_eval_cases

pytestmark = pytest.mark.gpu

#: worst device-vs-oracle 3-D IoU difference per match (test_gpu_track_gt.py), in 2^-32 cost units
IOU_BOUND = 2e-2 * 2.0 ** 32


def _run(tables, **kw):
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in tables.items() if k != 'sequences'}
    return evaluate.tracking_metrics(d['pred'], d['pred_id'], d['pred_cnt'], d['gt_box'], d['gt_obj'], d['gt_type'], d['gt_level'],
                                     d['gt_cnt'], d['num_frames'], d['n_obj'], **kw)


def _same(rec, ref):
    np.testing.assert_array_equal(rec[..., :4], ref[..., :4])
    assert (np.abs(rec[..., 4] - ref[..., 4]) <= ref[..., 0] * IOU_BOUND).all()


def _scene(seed, frames=14, objects=16):
    """one prepared sequence: objects of types 1, 2, 4 on straight paths (some crossing 30 m or 50 m), 20 % level-2 rows, objects
    absent from some frames, detections jittered with scores on a 0.01 grid offset by 0.005, misses, an id swap between two
    objects, a fragmented track, duplicates with their own ids and far false positives"""
    g = np.random.default_rng([seed, 0x7E1])
    dims = {1: (4.6, 2.0, 1.6), 2: (0.9, 0.9, 1.8), 4: (1.9, 0.8, 1.7)}
    typ = g.choice([1, 2, 4], objects)
    ang = g.uniform(-np.pi, np.pi, objects)
    rad = g.uniform(8.0, 70.0, objects)
    rad[:3] = [29.63, 49.57, 30.46]                              # straddlers
    vel = g.uniform(-0.25, 0.25, (objects, 2))
    vel[:3] = np.stack([np.cos(ang[:3]), np.sin(ang[:3])], 1) * np.array([0.1, 0.1, -0.1])[:, None]
    present = g.random((objects, frames)) < 0.9
    next_id = 1000
    seq = []
    for f in range(frames):
        preds, gts = [], []
        for o in range(objects):
            if not present[o, f]:
                continue
            c = np.array([rad[o] * np.cos(ang[o]), rad[o] * np.sin(ang[o])]) + vel[o] * f
            b = [c[0], c[1], -1.0, *dims[typ[o]], ang[o] + 0.02 * f]
            gts.append((b, int(typ[o]), 2 if g.random() < 0.2 else 1, o))
            if g.random() < 0.12:
                continue                                         # a miss
            pid = 100 + o
            if o in (3, 4) and f >= frames // 2:
                pid = 100 + (7 - o)                              # objects 3 and 4 swap ids
            if o == 5 and f >= frames // 3:
                pid = 500                                        # a fragment
            j = g.normal(0, 0.04, 3)
            pb = [b[0] + j[0], b[1] + j[1], b[2], b[3] * (1 + j[2]), b[4], b[5], b[6] + g.normal(0, 0.02)]
            preds.append((pb, np.floor(g.uniform(0.02, 0.98) * 100) / 100 + 0.005, int(typ[o]), pid))
            if g.random() < 0.12:
                d = list(pb)
                d[0] += g.choice([-0.35, 0.3])
                preds.append((d, np.floor(g.uniform(0.02, 0.98) * 100) / 100 + 0.005, int(typ[o]), next_id))
                next_id += 1
        for _ in range(2):
            t = int(g.choice([1, 2, 4]))
            a = g.uniform(-np.pi, np.pi)
            preds.append(([90 * np.cos(a), 90 * np.sin(a), -1.0, *dims[t], a], np.floor(g.uniform(0.02, 0.98) * 100) / 100 + 0.005,
                          t, next_id))
            next_id += 1
        seq.append(track_eval_cases.frame(preds, gts))
    return seq


@pytest.fixture(scope='module')
def scenes():
    return [_scene(s) for s in (1, 2, 3)]


def test_device_matches_oracle(scenes):
    ref, margin = track_eval_ref.records(scenes)
    assert margin.value > 1e-5, (margin.value, margin.where)
    rec, d = _run(track_eval_cases.pad_sequences(scenes), breakdowns=('object', 'range'))
    _same(rec, ref)
    assert ref[[0, 1, 3], 1, 0, 3].sum() > 0 and ref[:4, 1, 0, 2].sum() > 0 and ref[:4, 1, 0, 1].sum() > 0
    assert ref[:4, 1, 0, 0].sum() > ref[:4, 0, 0, 0].sum() and ref[4:, 0, 0, 0].reshape(4, 3)[:, 1].any()
    want = track_eval_ref.mot_dict(ref, ('object', 'range'))
    for k, v in want.items():
        assert abs(d[k][0] - v[0]) <= (IOU_BOUND / 2.0 ** 32 if k.endswith('MOTP') else 0.0), (k, d[k], v)


@pytest.mark.parametrize('name', sorted(track_eval_cases.CASES))
def test_hand_case_device(name):
    seqs, breakdowns, check = track_eval_cases.CASES[name]()
    ref, _ = track_eval_ref.records(seqs)
    rec, _ = _run(track_eval_cases.pad_sequences(seqs), breakdowns=('object', 'range'))
    _same(rec, ref)
    check(rec, evaluate.mot_dict(rec, breakdowns))
    obj, d = _run(track_eval_cases.pad_sequences(seqs), breakdowns=('object',))    # shards outside the breakdowns stay 0
    np.testing.assert_array_equal(obj[:4], rec[:4])
    assert not obj[4:].any() and d == evaluate.mot_dict(rec, ('object',))


def test_large_component():
    """40 pedestrian predictions on a chain of 30 overlapping pedestrians 0.3 m apart over three frames: one component per frame,
    run by the whole block"""
    g = np.random.default_rng(11)
    frames = []
    for f in range(3):
        gts, preds = [], []
        for i in range(30):
            size = tuple(np.array([1.0, 1.0, 1.8]) * g.uniform(0.95, 1.05, 3))
            gts.append((track_eval_cases.box(0.3 * i + 10.0 + 0.02 * f, 1.0, g.uniform(-0.02, 0.02), size), 2, 1 + int(g.random() < 0.3), i))
        for i in range(40):
            x = 10.0 + 0.02 * f + (0.15 + 0.3 * i if i < 29 else 0.3 * g.integers(0, 30) + g.uniform(-0.08, 0.08))
            size = tuple(np.array([1.0, 1.0, 1.8]) * g.uniform(0.95, 1.05, 3))
            pid = i if f < 2 or i % 3 else 100 + i
            preds.append((track_eval_cases.box(x, 1.0 + g.uniform(-0.05, 0.05), g.uniform(-0.3, 0.3), size),
                          0.005 + 0.02 * i + 0.01 * (i % 2), 2, pid))
        frames.append(track_eval_cases.frame(preds, gts))
    ref, margin = track_eval_ref.records([frames])
    assert margin.value > 1e-5, (margin.value, margin.where)
    rec, _ = _run(track_eval_cases.pad_sequences([frames]), breakdowns=('object', 'range'))
    _same(rec, ref)
    assert ref[1, 1, 0, 0] > 40 and ref[1, 1, 0, 3] > 0


def test_deterministic_and_batched(scenes):
    t = track_eval_cases.pad_sequences(scenes)
    whole, _ = _run(t, breakdowns=('object', 'range'))
    again, _ = _run(t, breakdowns=('object', 'range'))
    np.testing.assert_array_equal(whole, again)
    alone = sum(_run(track_eval_cases.pad_sequences([s]), breakdowns=('object', 'range'))[0] for s in scenes)
    np.testing.assert_array_equal(alone, whole)


def test_duplicate_ids_and_capacity_raise():
    b = track_eval_cases.box
    dup = [[track_eval_cases.frame([(b(5.0), 0.5, 1, 3), (b(-5.0), 0.5, 2, 3)], [(b(5.0), 1, 1, 0)])]]
    with pytest.raises(ValueError, match='share an id'):
        _run(track_eval_cases.pad_sequences(dup))
    dup_gt = [[track_eval_cases.frame([], [(b(5.0), 1, 1, 0), (b(-5.0), 1, 1, 0)])]]
    with pytest.raises(ValueError, match='share an id'):
        _run(track_eval_cases.pad_sequences(dup_gt))
    seqs, _, _ = track_eval_cases.CASES['retention']()
    with pytest.raises(RuntimeError, match='max_pairs'):
        _run(track_eval_cases.pad_sequences(seqs), max_pairs=2)


def _sequences(seeds, frames=16):
    seqs = []
    for seed in seeds:
        s = synthetic.synthetic_sequence(seed, frames=frames, tracks=16, n_background=500, ego_step=0.5, max_speed=0.3, radius=80.0)
        infos = synthetic.synthetic_ground_truth(s, seed, name='seq%d' % seed)
        boxes, counts, _ = synthetic.detections_from_sequence(s, seed)
        seqs.append((s, infos, boxes, counts))
    names = ['seq%d' % seed for seed in seeds]
    gt = ground_truth_from_infos(sum([sc[1] for sc in seqs], []), names)
    res = track_sequences(torch.from_numpy(np.stack([sc[2] for sc in seqs])).cuda(), torch.from_numpy(np.stack([sc[3] for sc in seqs])),
                          torch.from_numpy(np.stack([sc[0]['poses'] for sc in seqs])), max_entries=1 << 20)
    return seqs, names, gt, res


def test_evaluate_tracks_matches_frame_dicts():
    """evaluate_tracks on a track_sequences result equals the estimator on convert_frame_format's frames of its to_reference
    tracks (lidar boxes by the oracle's transform_boxes3d(inverse=True))"""
    seqs, names, gt, res = _sequences((5, 6))
    tracks, _ = res.to_reference(names, gt.frame_ids)
    preds, infos = [], []
    for i, (_, sinfos, _, _) in enumerate(seqs):
        for f, info in enumerate(sinfos):
            fid = gt.frame_ids[i][f]
            ids, rows, score, name = [], [], [], []
            for tid, t in tracks[names[i]].items():
                for j, sid in enumerate(t['sample_idx']):
                    if str(sid) == fid:
                        ids.append(tid)
                        rows.append(track_gt_ref.lidar_boxes(t['boxes_global'][[j]], t['pose'][j])[0])
                        score.append(t['score'][j])
                        name.append(t['name'][j])
            preds.append({'sequence_name': names[i], 'frame_id': f, 'obj_ids': np.array(ids, np.int64),
                          'boxes_lidar': np.array(rows, np.float32).reshape(-1, 7), 'score': np.array(score, np.float32),
                          'name': np.array(name)})
            infos.append(info)
    for cfg in (['object'], ['object', 'range']):
        d, rec = evaluate.evaluate_tracks(res, gt, CLASS_NAMES, cfg, return_records=True)
        est = evaluate.WaymoTrackingMetricsEstimator()
        want = est.waymo_evaluation(preds, infos, CLASS_NAMES, config_type=cfg, distance_thresh=1000, fake_gt_infos=False)
        _same(rec, est.records)
        assert rec[:4, 1, 0, 0].sum() > 0 and set(d) == set(want)
        for k, v in want.items():
            assert abs(d[k][0] - v[0]) <= (IOU_BOUND / 2.0 ** 32 if k.endswith('MOTP') else 0.0), (k, d[k], v)


def test_evaluate_offboard_tracking_matches_frame_dicts():
    """evaluate_offboard_tracking on refine_sequence results equals the estimator on their to_reference frames without the dropped
    detections"""
    seqs, names, gt, res = _sequences((5, 6))
    models = synthetic.refine_models(5)
    results = []
    with torch.no_grad():
        for i, (s, _, _, _) in enumerate(seqs):
            results.append(offboard.refine_sequence(torch.from_numpy(s['frames']).cuda(), s['frame_offsets'],
                                                    torch.from_numpy(s['poses']).cuda(), res, models, sequence=i))
    d, rec = evaluate.evaluate_offboard_tracking(results, gt, CLASS_NAMES, ['object', 'range'], return_records=True)
    preds, infos = [], []
    for i, (_, sinfos, _, _) in enumerate(seqs):
        got = {x['frame_id']: x for x in results[i].to_reference(names[i], range(len(sinfos)))}
        for f, info in enumerate(sinfos):
            x = got.get(f)
            if x is None:
                x = {'sequence_name': names[i], 'obj_ids': np.zeros(0, np.int64), 'boxes_lidar': np.zeros((0, 7), np.float32),
                     'score': np.zeros(0, np.float32), 'name': np.array([])}
            n = len(x['obj_ids'])
            preds.append({'sequence_name': names[i], 'obj_ids': x['obj_ids'], 'boxes_lidar': x['boxes_lidar'][:n],
                          'score': x['score'][:n], 'name': x['name'][:n]})
            infos.append(info)
    est = evaluate.WaymoTrackingMetricsEstimator()
    want = est.waymo_evaluation(preds, infos, CLASS_NAMES, config_type=['object', 'range'], fake_gt_infos=False)
    _same(rec, est.records)
    assert rec[:4, 1, 0, 0].sum() > 0
    for k, v in want.items():
        assert abs(d[k][0] - v[0]) <= (IOU_BOUND / 2.0 ** 32 if k.endswith('MOTP') else 0.0), (k, d[k], v)

"""detzero_b200.evaluate (csrc/det_eval.cu) against the numpy restatement oracle/det_eval_ref.py: the int64 records (TP, FP, FN,
TPH) exactly and the AP dicts equal, on synthetic scenes whose every decision the oracle takes at least 1e-5 from its threshold, on
the hand-computed cases, on one large assignment component; records add up over frame sets and do not depend on the run or the
chunking; the full offboard chain scored on the device equals the reference-shaped entry point on the same frames."""
import numpy as np
import pytest
import torch

from detzero_b200 import evaluate, offboard, synthetic
from detzero_b200.track import CLASS_NAMES, ground_truth_from_infos, track_sequences
from oracle import det_eval_ref
from tests import det_eval_cases

pytestmark = pytest.mark.gpu


def _dev(tables):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in tables.items()}


def _scene(seed, frames=6, tracks=24):
    """frame dicts (predictions, ground-truth annos) of a synthetic sequence: difficulty 2 on some rows, objects 6 to 70 m out,
    detections with scores on a 0.01 grid offset by 0.005, injected duplicates, pi-flipped headings, and pairs straddling the
    30 m and 50 m range boundaries"""
    g = np.random.default_rng([seed, 0xE7A])
    s = synthetic.synthetic_sequence(seed, frames=frames, tracks=tracks, n_background=100, radius=70.0)
    diff = [[2 if g.random() < 0.2 else 0 for _ in range(200)] for _ in range(tracks)]
    gts = [i['annos'] for i in synthetic.synthetic_ground_truth(s, seed, name='seq%d' % seed, difficulty=diff)]
    boxes, counts, _ = synthetic.detections_from_sequence(s, seed, fp=4)
    preds = []
    for f in range(frames):
        rows = boxes[f, :counts[f]].copy()
        flip = g.random(len(rows)) < 0.15
        rows[flip, 6] = np.where(rows[flip, 6] > 0, rows[flip, 6] - np.pi, rows[flip, 6] + np.pi)
        dup = rows[g.random(len(rows)) < 0.2].copy()
        dup[:, 0] += np.where(g.random(len(dup)) < 0.5, 0.12, -0.2)
        rows = np.concatenate([rows, dup])
        rows[:, 7] = g.uniform(0.02, 0.98, len(rows))
        extra_gt, extra_pred = [], []
        for r, a in ((29.97, 30.03), (49.96, 50.04), (30.04, 29.98)):
            ang = g.uniform(-np.pi, np.pi)
            c, sn = np.cos(ang), np.sin(ang)
            extra_gt.append([r * c, r * sn, -1.0, 4.5, 1.9, 1.6, ang])
            extra_pred.append([a * c, a * sn, -1.0, 4.5, 1.9, 1.6, ang + 0.05, g.uniform(0.02, 0.98), 1])
        rows = np.concatenate([rows, np.array(extra_pred, np.float32)])
        rows[:, 7] = np.floor(rows[:, 7] * 100) / 100 + 0.005
        preds.append({'boxes_lidar': rows[:, :7].astype(np.float32), 'score': rows[:, 7].astype(np.float32),
                      'name': np.array([CLASS_NAMES[int(c) - 1] for c in rows[:, 8]])})
        a = dict(gts[f])
        n = len(extra_gt)
        a['gt_boxes_lidar'] = np.concatenate([a['gt_boxes_lidar'], np.array(extra_gt, np.float32)])
        a['name'] = np.concatenate([a['name'], np.array(['Vehicle'] * n)])
        a['difficulty'] = np.concatenate([a['difficulty'], np.array([0, 2, 1][:n], np.int32)])
        a['num_points_in_gt'] = np.concatenate([a['num_points_in_gt'], np.array([40, 3, 12][:n], np.int32)])
        gts[f] = a
    return preds, gts


@pytest.fixture(scope='module')
def scenes():
    preds, gts = [], []
    for seed in (1, 2, 3):
        p, g = _scene(seed)
        preds += p
        gts += g
    return preds, gts


@pytest.mark.parametrize('box_type', ['3d', 'bev'])
def test_device_matches_oracle(scenes, box_type):
    preds, gts = scenes
    cfg = ['object', 'range', box_type]
    ref_ap, ref_rec, margin = det_eval_ref.waymo_evaluation(preds, gts, CLASS_NAMES, cfg, 1000, False)
    assert margin.value > 1e-5, (margin.value, margin.where)
    est = evaluate.WaymoDetectionMetricsEstimator()
    ap = est.waymo_evaluation(preds, gts, CLASS_NAMES, config_type=cfg, distance_thresh=1000, fake_gt_infos=False)
    np.testing.assert_array_equal(est.records, ref_rec)
    assert ap == ref_ap
    assert ref_rec[:, 1, 0, 0].sum() > ref_rec[:, 0, 0, 0].sum() > 0 and ref_rec[4:, 0, 0, 0].reshape(4, 3)[0].all()


@pytest.mark.parametrize('name', sorted(det_eval_cases.CASES))
def test_hand_case_device(name):
    frames, breakdowns, check = det_eval_cases.CASES[name]()
    for box_type in ('3d', 'bev'):
        rec, ap = evaluate.detection_metrics(**_dev(det_eval_cases.pad_frames(frames)), box_type=box_type, breakdowns=breakdowns)
        ref, _ = det_eval_ref.records(frames, box_type, breakdowns)
        np.testing.assert_array_equal(rec, ref)
        check(rec, ap)


def test_large_component():
    """40 pedestrian predictions on a chain of 30 overlapping pedestrians 0.3 m apart: one component, solved by the block"""
    g = np.random.default_rng(11)
    gts, preds = [], []
    for i in range(30):
        size = tuple(np.array([1.0, 1.0, 1.8]) * g.uniform(0.95, 1.05, 3))
        gts.append((det_eval_cases.box(0.3 * i + 10.0, 1.0, g.uniform(-0.02, 0.02), size), 2, 1 + int(g.random() < 0.3)))
    for i in range(40):
        x = 10.0 + (0.15 + 0.3 * i if i < 29 else 0.3 * g.integers(0, 30) + g.uniform(-0.08, 0.08))
        size = tuple(np.array([1.0, 1.0, 1.8]) * g.uniform(0.95, 1.05, 3))
        preds.append((det_eval_cases.box(x, 1.0 + g.uniform(-0.05, 0.05), g.uniform(-0.3, 0.3), size), 0.005 + 0.02 * i + 0.01 * (i % 2), 2))
    frames = [det_eval_cases.frame(preds, gts)]
    for box_type in ('3d', 'bev'):
        ref, margin = det_eval_ref.records(frames, box_type, ('object', 'range'))
        assert margin.value > 1e-5, (margin.value, margin.where)
        rec, _ = evaluate.detection_metrics(**_dev(det_eval_cases.pad_frames(frames)), box_type=box_type, breakdowns=('object', 'range'))
        np.testing.assert_array_equal(rec, ref)
        assert ref[1, 1, 0, 0] > 20


def test_additive_and_deterministic(scenes):
    preds, gts = scenes
    t = evaluate.frame_tables(preds, gts, CLASS_NAMES, 1000, False)
    d = _dev(t)
    run = lambda sl, **kw: evaluate.detection_metrics(*(d[k][sl] for k in ('pred', 'pred_cnt', 'gt_box', 'gt_type', 'gt_level', 'gt_cnt')),
                                                     breakdowns=('object', 'range'), **kw)[0]
    whole = run(slice(None))
    assert whole.any()
    np.testing.assert_array_equal(run(slice(None, 7)) + run(slice(7, None)), whole)
    np.testing.assert_array_equal(run(slice(None)), whole)
    np.testing.assert_array_equal(run(slice(None), frame_chunk=5), whole)
    np.testing.assert_array_equal(run(slice(None), frame_chunk=1), whole)


def test_max_pairs_capacity():
    frames, breakdowns, _ = det_eval_cases.CASES['contention']()
    with pytest.raises(RuntimeError, match='max_pairs'):
        evaluate.detection_metrics(**_dev(det_eval_cases.pad_frames(frames)), max_pairs=2)


def test_offboard_chain():
    """track_sequences -> refine_sequence -> evaluate_offboard equals waymo_evaluation on the same frames in frame-dict form"""
    seqs = []
    for seed in (5, 6):
        s = synthetic.synthetic_sequence(seed, frames=16, tracks=16, n_background=500, ego_step=0.5, max_speed=0.3, radius=80.0)
        infos = synthetic.synthetic_ground_truth(s, seed, name='seq%d' % seed)
        boxes, counts, _ = synthetic.detections_from_sequence(s, seed)
        seqs.append((s, infos, boxes, counts))
    names = ['seq5', 'seq6']
    gt = ground_truth_from_infos(sum([sc[1] for sc in seqs], []), names)
    res = track_sequences(torch.from_numpy(np.stack([sc[2] for sc in seqs])).cuda(), torch.from_numpy(np.stack([sc[3] for sc in seqs])),
                          torch.from_numpy(np.stack([sc[0]['poses'] for sc in seqs])), max_entries=1 << 20)
    models = synthetic.refine_models(5)
    results = []
    with torch.no_grad():
        for i, (s, _, _, _) in enumerate(seqs):
            results.append(offboard.refine_sequence(torch.from_numpy(s['frames']).cuda(), s['frame_offsets'],
                                                    torch.from_numpy(s['poses']).cuda(), res, models, sequence=i))
    for cfg, dist in ((['object', '3d'], 40), (['object', 'range', 'bev'], 60)):
        ap, rec = evaluate.evaluate_offboard(results, gt, CLASS_NAMES, cfg, dist, return_records=True)
        assert rec[:4, 1, 0, 0].sum() + rec[:4, 1, 0, 2].sum() > 0 and rec[:4, 1, 0, 0].sum() + rec[:4, 1, 0, 1].sum() > 0
        preds, annos = [], []
        for i, (s, infos, _, _) in enumerate(seqs):
            got = {d['frame_id']: d for d in results[i].to_reference(names[i], range(len(infos)))}
            for f, info in enumerate(infos):
                preds.append(got.get(f, {'sequence_name': names[i], 'frame_id': f, 'boxes_lidar': np.array([]).reshape(0, 7),
                                         'score': np.array([]), 'name': np.array([])}))
                annos.append(info['annos'])
        want = evaluate.WaymoDetectionMetricsEstimator().waymo_evaluation(preds, annos, CLASS_NAMES, config_type=cfg,
                                                                          distance_thresh=dist, fake_gt_infos=False)
        assert ap == want

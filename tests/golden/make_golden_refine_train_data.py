"""Golden vectors for the refiner training samples (tests/golden/refine_train_data.npz), produced by the reference's OWN code on the
CPU: WaymoGeometryDataset / WaymoConfidenceDataset.extract_track_feature with training = True (and augment_single = True for the
GRM, so geometry_augment.augment_single_box runs), __init__ bypassed, on the four-track sequence of make_golden_refine_data.py.

Ground truth: the boxes of each track moved and resized a little, as float32 world boxes; tracks 0 and 3 have unmatched slots.
The CRM's refine_iou is a synthetic label per box, uniform on [0, 1] (so on both sides of 0.25 and 0.5).

Every random draw of the training branch is replaced, in the dataset and augment modules' namespaces, by a stub that hands out the
oracle's keyed draws (oracle/refine_train_data_ref.py train_draw) in the reference's call order: random.randint (kept count),
random.sample (kept boxes), np.random.choice (GRM queries), np.random.randint (CRM init box) and np.random.random (GRM flips).
sample_points is replaced as make_golden_refine_data.py replaces it, so the features can be compared row by row.

    python tests/golden/make_golden_refine_train_data.py /path/to/reference
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

SEED, EPOCH = 7, 3
MEM_STRIDE = 8          # every 8th GRM memory row is stored
UNMATCHED = {0: np.arange(3, 200, 7), 3: np.array([2, 5])}


def targets(s):
    """(gt_boxes (B, L, 7) f64 holding float32 values, matched (B, L) u8, iou (B, L) f32) of the golden sequence"""
    g = np.random.default_rng(123)
    B, L = s['boxes'].shape[:2]
    gt = s['boxes'].copy()
    gt[..., :3] += g.normal(0, 0.1, (B, L, 3))
    gt[..., 3:6] *= g.uniform(0.9, 1.1, (B, L, 3))
    gt[..., 6] += g.normal(0, 0.05, (B, L))
    matched = np.zeros((B, L), np.uint8)
    for b, n in enumerate(s['box_num']):
        matched[b, :int(n)] = 1
        if b in UNMATCHED:
            matched[b, UNMATCHED[b]] = 0
    gt[matched == 0] = 0
    iou = np.where(np.arange(L)[None, :] < np.asarray(s['box_num'])[:, None], g.uniform(0, 1, (B, L)), 0)
    return gt.astype(np.float32).astype(np.float64), matched, iou.astype(np.float32)


def main(ref):
    import ref_import
    ref_import.REF = ref
    ref_import.install()
    ref_import._pkg('detzero_refine.datasets', ref + '/refining/detzero_refine/datasets')
    ref_import._pkg('detzero_refine.datasets.waymo', ref + '/refining/detzero_refine/datasets/waymo')
    from detzero_refine.datasets.waymo import waymo_confidence_dataset as crm_mod
    from detzero_refine.datasets.waymo import waymo_geometry_dataset as grm_mod
    from detzero_refine.utils import geometry_augment as aug_mod
    from make_golden_refine_data import sequence
    from oracle import refine_data_ref as R
    from oracle import refine_train_data_ref as T

    s = sequence()
    gt, matched, iou = targets(s)
    q = {k: [] for k in ('randint', 'sample', 'choice', 'np_randint', 'random', 'points')}

    def pop(name, *check):
        v, want = q[name].pop(0)
        assert tuple(want) == tuple(check), (name, want, check)
        return v

    def fake_sample_points(pts, sample_num=4096, replace=False):
        sel = q['points'].pop(0)
        assert len(sel) == min(len(pts), sample_num), (len(sel), len(pts), sample_num)
        if len(pts) >= sample_num:
            return pts[sel]
        return np.concatenate((pts, np.zeros((sample_num - len(pts), pts.shape[1]), dtype=np.float32)), axis=0)

    fake_random = types.SimpleNamespace(randint=lambda a, b: pop('randint', a, b),
                                        sample=lambda pop_, k: pop('sample', len(pop_), k))
    fake_np = types.ModuleType('numpy')
    fake_np.__dict__.update(np.__dict__)
    fake_np.random = types.SimpleNamespace(choice=lambda n, k, replace=True: pop('choice', n, k, replace),
                                           randint=lambda lo, hi=None: pop('np_randint', lo, hi),
                                           random=lambda: pop('random'))
    for mod in (grm_mod, crm_mod):
        mod.sample_points = fake_sample_points
        mod.random = fake_random
        mod.np = fake_np
    aug_mod.np = fake_np

    def dataset(cls, encoding, qn, kq, km=None):
        d = cls.__new__(cls)
        d.training, d.encoding, d.query_num, d.query_pts_num = True, encoding, qn, kq
        if km is not None:
            d.memory_pts_num = km
        d.class_map = {'Vehicle': 1, 'Pedestrian': 2, 'Cyclist': 3, 1: 'Vehicle', 2: 'Pedestrian', 3: 'Cyclist'}
        d.augment_single, d.augment_full = True, False
        return d

    names = {1: 'Vehicle', 2: 'Pedestrian', 3: 'Cyclist'}
    out = {k: s[k] for k in ('frame_offsets', 'poses', 'boxes', 'frame_of_box', 'scores', 'box_num', 'cls', 'track_uid')}
    out['points'] = s['frames'][:, 1:5]
    out['gt_boxes'], out['matched'], out['iou'] = gt, matched, iou
    out['seed'], out['epoch'] = np.int64(SEED), np.int64(EPOCH)
    for b, L in enumerate(s['box_num']):
        L = int(L)
        bx, sc, fob = s['boxes'][b], s['scores'][b], s['frame_of_box'][b]
        crops = R.track_crops(s['frames'], s['frame_offsets'], s['poses'], bx, fob, L)
        uid = int(s['track_uid'][b])
        mt = matched[b, :L].astype(bool)
        info = {'sequence_name': 'seq', 'obj_id': str(b), 'name': names[int(s['cls'][b])], 'boxes_global': bx[:L].astype(np.float32),
                'score': sc[:L].copy(), 'sample_idx': np.arange(L), 'pose': s['poses'][fob[:L]], 'matched': mt,
                'matched_tracklet': True, 'state': 'dynamic', 'gt_boxes_global': gt[b, :L].astype(np.float32),
                'refine_iou': iou[b, :L].copy()}
        pts = [np.concatenate([c[:, :3] + bx[j, :3], c[:, 3:4]], 1) for j, c in enumerate(crops)]          # world float64 rows

        # GRM: randint, sample, choice, random per kept box, sample_points (memory, then each query)
        o = T.geometry_train_track(crops, bx, sc, gt[b], matched[b], L, uid, SEED, EPOCH)
        elig = np.nonzero(mt)[0]
        m, n = len(elig), len(o['kept'])
        q['randint'].append((n, (min(5, m), m)))
        q['sample'].append((list(np.searchsorted(elig, o['kept'])), (m, n)))
        q['choice'].append((np.asarray(o['query_slots']), (n, min(3, n), False)))
        q['random'].extend((0.25 if f else 0.75, ()) for f in o['flip'])
        q['points'].append(o['sel'][1])
        q['points'].extend(o['sel'][0])
        r = dataset(grm_mod.WaymoGeometryDataset, ['xyz', 'intensity', 'p2s', 'score'], 3, 256, 4096).extract_track_feature(
            dict(info, pts=[p.copy() for p in pts]))
        assert not any(q.values()), {k: len(v) for k, v in q.items()}
        out['grm_kept_%d' % b], out['grm_query_%d' % b], out['grm_flip_%d' % b] = o['kept'], o['query_slots'], o['flip']
        for k in ('geo_query_points', 'geo_query_boxes', 'gt_geo_query_boxes', 'geo_trajectory', 'gt_geo_trajectory'):
            out['grm_%s_%d' % (k, b)] = np.asarray(r[k], np.float32)
        out['grm_geo_memory_points_%d' % b] = np.asarray(r['geo_memory_points'], np.float32)[::MEM_STRIDE]
        out['grm_geo_query_num_%d' % b] = np.int64(r['geo_query_num'])

        # CRM: randint, sample, np.random.randint, sample_points per kept box
        o = T.confidence_train_track(crops, bx, sc, iou[b], L, uid, SEED, EPOCH)
        n = len(o['kept'])
        q['randint'].append((n, (min(5, L), L)))
        q['sample'].append((list(o['kept']), (L, n)))
        q['np_randint'].append((o['init_slot'], (0, n)))
        q['points'].extend(o['sel'])
        r = dataset(crm_mod.WaymoConfidenceDataset, ['xyz', 'intensity', 'p2co', 'score'], 200, 256).extract_track_feature(
            dict(info, pts=[p.copy() for p in pts]))
        assert not any(q.values()), {k: len(v) for k, v in q.items()}
        # conf_points of a few kept positions (the first, the init box, the last) and the padding right after them
        keep = np.array(sorted({0, int(o['init_slot']), n - 1, min(n, 199)}))
        out['crm_kept_%d' % b], out['crm_init_%d' % b], out['crm_rows_%d' % b] = o['kept'], np.int64(o['init_slot']), keep
        out['crm_conf_points_%d' % b] = np.asarray(r['conf_points'], np.float32)[keep]
        out['crm_conf_score_%d' % b] = np.asarray(r['conf_score'], np.float32)
        out['crm_iou_%d' % b] = np.asarray(r['iou'], np.float32)
        out['crm_box_num_%d' % b] = np.int64(r['box_num'])
        print('track %d: L %d, GRM keeps %d of %d matched (%d flipped), CRM keeps %d, init %d' % (
            b, L, len(out['grm_kept_%d' % b]), m, int(out['grm_flip_%d' % b].sum()), n, o['init_slot']))
    np.savez_compressed(os.path.join(HERE, 'refine_train_data.npz'), **out)


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else '/root/reference')

"""Golden vectors for the PRM training samples (tests/golden/prm_train_data.npz), produced by the reference's OWN code on the CPU:
WaymoPositionDataset.extract_track_feature with training = True and augment_full = False, __init__ bypassed, on the four-track
sequence and ground truth of make_golden_refine_train_data.py (tracks 0 and 3 have unmatched slots).

Every random draw of the training branch is replaced, in the dataset module's namespace, by a stub that hands out the draws of the
restatement (tests/prm_train_data_ref.py position_train_track) in the reference's call order: random.randint (kept count),
random.sample (kept boxes, handed out in ascending order) and np.random.randint (init box).  sample_points is replaced as
make_golden_refine_data.py replaces it (query, then memory, per kept box), so the features can be compared row by row.

    python tests/golden/make_golden_prm_train_data.py /path/to/reference
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)


def main(ref):
    import ref_import
    ref_import.REF = ref
    ref_import.install()
    ref_import._pkg('detzero_refine.datasets', ref + '/refining/detzero_refine/datasets')
    ref_import._pkg('detzero_refine.datasets.waymo', ref + '/refining/detzero_refine/datasets/waymo')
    from detzero_refine.datasets.waymo import waymo_position_dataset as prm_mod
    from make_golden_refine_data import sequence
    from make_golden_refine_train_data import EPOCH, SEED, targets
    from oracle import refine_data_ref as R
    from tests import prm_train_data_ref as PT

    s = sequence()
    gt, matched, _ = targets(s)
    q = {k: [] for k in ('randint', 'sample', 'np_randint', 'points')}

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

    fake_np = types.ModuleType('numpy')
    fake_np.__dict__.update(np.__dict__)
    fake_np.random = types.SimpleNamespace(randint=lambda lo, hi=None: pop('np_randint', lo, hi))
    prm_mod.sample_points = fake_sample_points
    prm_mod.random = types.SimpleNamespace(randint=lambda a, b: pop('randint', a, b), sample=lambda pop_, k: pop('sample', len(pop_), k))
    prm_mod.np = fake_np

    d = prm_mod.WaymoPositionDataset.__new__(prm_mod.WaymoPositionDataset)
    d.training, d.encoding, d.query_num, d.query_pts_num, d.memory_pts_num = True, ['xyz', 'intensity', 'p2co', 'score'], 200, 256, 48
    d.class_map = {'Vehicle': 1, 'Pedestrian': 2, 'Cyclist': 3, 1: 'Vehicle', 2: 'Pedestrian', 3: 'Cyclist'}
    d.augment_single, d.augment_full = False, False

    names = {1: 'Vehicle', 2: 'Pedestrian', 3: 'Cyclist'}
    out = {k: s[k] for k in ('frame_offsets', 'poses', 'boxes', 'frame_of_box', 'scores', 'box_num', 'cls', 'track_uid')}
    out['points'] = s['frames'][:, 1:5]
    out['gt_boxes'], out['matched'] = gt, matched
    out['seed'], out['epoch'] = np.int64(SEED), np.int64(EPOCH)
    for b, L in enumerate(s['box_num']):
        L = int(L)
        bx, sc, fob = s['boxes'][b], s['scores'][b], s['frame_of_box'][b]
        crops = R.track_crops(s['frames'], s['frame_offsets'], s['poses'], bx, fob, L)
        uid = int(s['track_uid'][b])
        mt = matched[b, :L].astype(bool)
        info = {'sequence_name': 'seq', 'obj_id': str(b), 'name': names[int(s['cls'][b])], 'boxes_global': bx[:L].astype(np.float32),
                'score': sc[:L].copy(), 'sample_idx': np.arange(L), 'pose': s['poses'][fob[:L]], 'matched': mt,
                'matched_tracklet': True, 'state': 'dynamic', 'gt_boxes_global': gt[b, :L].astype(np.float32)}
        pts = [np.concatenate([c[:, :3] + bx[j, :3], c[:, 3:4]], 1) for j, c in enumerate(crops)]          # world float64 rows

        o = PT.position_train_track(crops, bx, sc, gt[b], matched[b], L, uid, SEED, EPOCH)
        elig = np.nonzero(mt)[0]
        m, n = len(elig), len(o['kept'])
        q['randint'].append((n, (min(5, m), m)))
        q['sample'].append((list(np.searchsorted(elig, o['kept'])), (m, n)))
        q['np_randint'].append((o['init_slot'], (0, n)))
        for sq, sm in zip(*o['sel']):
            q['points'].extend([sq, sm])
        r = d.extract_track_feature(dict(info, pts=[p.copy() for p in pts]))
        assert not any(q.values()), {k: len(v) for k, v in q.items()}
        # the features of a few kept positions (the first, the init box, the last) and the padding right after them
        keep = np.array(sorted({0, int(o['init_slot']), n - 1, min(n, 199)}))
        out['prm_kept_%d' % b], out['prm_init_%d' % b], out['prm_rows_%d' % b] = o['kept'], np.int64(o['init_slot']), keep
        out['prm_pos_query_points_%d' % b] = np.asarray(r['pos_query_points'], np.float32)[keep]
        out['prm_pos_memory_points_%d' % b] = np.asarray(r['pos_memory_points'], np.float32)[keep]
        for k in ('pos_trajectory', 'gt_pos_trajectory', 'pos_init_box', 'padding_mask'):
            out['prm_%s_%d' % (k, b)] = np.asarray(r[k], np.float32)
        out['prm_box_num_%d' % b] = np.int64(r['box_num'])
        print('track %d: L %d, PRM keeps %d of %d matched, init %d' % (b, L, n, m, o['init_slot']))
    np.savez_compressed(os.path.join(HERE, 'prm_train_data.npz'), **out)


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else '/root/reference')

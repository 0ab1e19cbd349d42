"""Golden vectors for the refiner input builder (tests/golden/refine_data.npz), produced by the reference's OWN code on the CPU:
WaymoPositionDataset / WaymoGeometryDataset / WaymoConfidenceDataset.extract_track_feature (eval branch, __init__ bypassed) and their
revert_to_each_frame, on the tracks of a seeded synthetic_sequence placed within about 100 m of the origin with float32 world boxes
(the reference's trajectory arithmetic is float32, so larger offsets would blur the comparison).

The per-object inputs are what daemon/prepare_object_data.py writes: each box's points as float64 world rows [x, y, z, tanh(i)], taken
from the oracle's crop.  sample_points is replaced, in each dataset module's namespace, by a wrapper that keeps the oracle's keyed
selections (oracle/refine_data_ref.py) in the reference's call order, so the features can be compared row by row.

    python tests/golden/make_golden_refine_data.py /path/to/reference
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

SEED = 7
LENGTHS = [200, 1, 2, 9]
CLS = [1, 2, 1, 3]


def sequence():
    from detzero_b200.synthetic import synthetic_sequence
    s = synthetic_sequence(SEED, frames=200, tracks=len(LENGTHS), n_background=8, max_pts=2600, origin=(40.0, -25.0, 0.5),
                           ego_step=0.2, max_speed=0.08, lengths=LENGTHS, cls=CLS)
    s['boxes'] = s['boxes'].astype(np.float32).astype(np.float64)            # float32 world boxes, as the reference requires
    return thin(s)


def thin(s, cap=8):
    """Keep the file small: every box keeps at most `cap` of its points (the first, in frame order), except one box of the long
    track in each of the point-count classes 48-255, 256-2048 and > 2048, which keeps all of its points.  Removing points keeps
    every remaining point clear of the enlarged faces, so crop membership stays unambiguous."""
    from oracle import refine_data_ref as R
    frames, off = s['frames'], s['frame_offsets']
    drop = np.zeros(len(frames), bool)
    for b, L in enumerate(LENGTHS):
        rows = [R.crop_box(np.concatenate([frames[off[f]:off[f + 1], 1:4], np.arange(off[f], off[f + 1])[:, None]], 1),
                           s['poses'][f], s['boxes'][b, j])[:, 3].astype(np.int64) for j, f in enumerate(s['frame_of_box'][b, :L])]
        n = np.array([len(r) for r in rows])
        whole = set()
        if b == 0:
            for lo, hi in ((48, 256), (256, 2049), (2049, 1 << 30)):
                cand = np.nonzero((n >= lo) & (n < hi))[0]
                assert len(cand), (lo, hi)
                whole.add(int(cand[0]))
        for j, r in enumerate(rows):
            if j not in whole:
                drop[r[cap:]] = True
    keep = ~drop
    s['frames'] = frames[keep]
    s['frame_offsets'] = np.concatenate([[0], np.cumsum([keep[off[f]:off[f + 1]].sum() for f in range(len(off) - 1)])]).astype(np.int64)
    return s


def main(ref):
    import ref_import
    ref_import.REF = ref
    ref_import.install()
    ref_import._pkg('detzero_refine.datasets', ref + '/refining/detzero_refine/datasets')
    ref_import._pkg('detzero_refine.datasets.waymo', ref + '/refining/detzero_refine/datasets/waymo')
    from detzero_refine.datasets.waymo import waymo_confidence_dataset as crm_mod
    from detzero_refine.datasets.waymo import waymo_geometry_dataset as grm_mod
    from detzero_refine.datasets.waymo import waymo_position_dataset as prm_mod
    from oracle import refine_data_ref as R

    s = sequence()
    queue = []

    def fake_sample_points(pts, sample_num=4096, replace=False):
        sel = queue.pop(0)
        assert len(sel) == min(len(pts), sample_num), (len(sel), len(pts), sample_num)
        if len(pts) >= sample_num:
            return pts[sel]
        return np.concatenate((pts, np.zeros((sample_num - len(pts), pts.shape[1]), dtype=np.float32)), axis=0)
    for mod in (prm_mod, grm_mod, crm_mod):
        mod.sample_points = fake_sample_points

    def dataset(cls, encoding, qn, kq, km=None):
        d = cls.__new__(cls)
        d.training, d.encoding, d.query_num, d.query_pts_num = False, encoding, qn, kq
        if km is not None:
            d.memory_pts_num = km
        d.class_map = {'Vehicle': 1, 'Pedestrian': 2, 'Cyclist': 3, 1: 'Vehicle', 2: 'Pedestrian', 3: 'Cyclist'}
        d.augment_full = d.augment_single = False
        return d

    def fresh(info, pts):          # extract_track_feature transforms its inputs in place
        return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in info.items()} | {'pts': [p.copy() for p in pts]}

    names = {1: 'Vehicle', 2: 'Pedestrian', 3: 'Cyclist'}
    out = {k: s[k] for k in ('frame_offsets', 'poses', 'boxes', 'frame_of_box', 'scores', 'box_num', 'cls', 'track_uid')}
    out['points'] = s['frames'][:, 1:5]                            # [x, y, z, tanh(i)]; the frame column follows from frame_offsets
    out['seed'] = np.int64(SEED)
    g = np.random.default_rng(99)
    for b, L in enumerate(s['box_num']):
        L = int(L)
        bx, sc, fob = s['boxes'][b], s['scores'][b], s['frame_of_box'][b]
        crops = R.track_crops(s['frames'], s['frame_offsets'], s['poses'], bx, fob, L)
        uid = int(s['track_uid'][b])
        info = {'sequence_name': 'seq', 'obj_id': str(b), 'name': names[int(s['cls'][b])], 'boxes_global': bx[:L].astype(np.float32),
                'score': sc[:L].copy(), 'sample_idx': np.arange(L), 'pose': s['poses'][fob[:L]], 'matched': np.ones(L, bool),
                'matched_tracklet': True, 'state': 'dynamic', 'gt_boxes_global': np.zeros((L, 7), np.float32),
                'refine_iou': np.zeros(L, np.float32)}
        info_pts = [np.concatenate([c[:, :3] + bx[j, :3], c[:, 3:4]], 1) for j, c in enumerate(crops)]   # world float64 rows
        out['counts_%d' % b] = cnt = np.array([len(c) for c in crops])
        # per-box feature rows are stored for a subset of the box slots to keep the file small: the first box, the padding right
        # after the track and, on the long track, one box per point-count class
        keep = {0, min(L, 199)}
        for lo, hi in ((0, 1), (1, 48), (48, 256), (256, 2049), (2049, 1 << 30)):
            keep |= set(np.nonzero((cnt >= lo) & (cnt < hi))[0][:1 if b == 0 else 0].tolist())
        out['keep_%d' % b] = keep = np.array(sorted(keep))
        for enc_name, encoding in (('prm', R_P2CO), ('prmc', R_P2CO + ['class'])):
            if enc_name == 'prmc' and int(s['cls'][b]) != 3:
                continue
            o = R.position_track(crops, bx, sc, L, s['cls'][b], uid, SEED, with_class=enc_name == 'prmc')
            for q, m in zip(*o['sel']):
                queue.extend([q, m])
            r = dataset(prm_mod.WaymoPositionDataset, encoding, 200, 256, 48).extract_track_feature(
                fresh(info, info_pts))
            assert not queue
            for k in ('pos_query_points', 'pos_memory_points', 'pos_trajectory', 'padding_mask', 'pos_init_box'):
                v = np.asarray(r[k], np.float32)
                out['%s_%s_%d' % (enc_name, k, b)] = v[keep] if k in ('pos_query_points', 'pos_memory_points') else v
            if enc_name == 'prm':
                out['prm_sel_q_%d' % b] = np.concatenate(o['sel'][0])
                out['prm_sel_m_%d' % b] = np.concatenate(o['sel'][1])
                pred = np.concatenate([g.normal(0, 3, (L, 3)), bx[:L, 3:6] * g.uniform(0.9, 1.1, (L, 3)), g.uniform(-np.pi, np.pi, (L, 1))], 1)
                pred = pred.astype(np.float32)
                rl, _, rw, _ = dataset(prm_mod.WaymoPositionDataset, encoding, 200, 256, 48).revert_to_each_frame(
                    {'pred_boxes': [pred.copy()], 'pos_init_box': [r['pos_init_box']], 'pose': [info['pose']],
                     'gt_pos_trajectory': [np.zeros((L, 7), np.float32)]})
                out['prm_pred_%d' % b], out['prm_revert_lidar_%d' % b], out['prm_revert_world_%d' % b] = pred, rl[0], rw[0]
        o = R.confidence_track(crops, bx, sc, L, uid, SEED)
        queue.extend(o['sel'])
        r = dataset(crm_mod.WaymoConfidenceDataset, R_P2CO, 200, 256).extract_track_feature(fresh(info, info_pts))
        assert not queue
        out['crm_conf_points_%d' % b] = np.asarray(r['conf_points'], np.float32)[keep]
        out['crm_conf_score_%d' % b] = np.asarray(r['conf_score'], np.float32)
        out['crm_sel_%d' % b] = np.concatenate(o['sel'])
        o = R.geometry_track(crops, bx, sc, L, uid, SEED)
        queue.append(o['sel'][1])
        queue.extend(o['sel'][0])
        r = dataset(grm_mod.WaymoGeometryDataset, ['xyz', 'intensity', 'p2s', 'score'], 3, 256, 4096).extract_track_feature(
            fresh(info, info_pts))
        assert not queue
        for k in ('geo_query_points', 'geo_query_boxes'):
            out['grm_%s_%d' % (k, b)] = np.asarray(r[k], np.float32)
        out['grm_geo_memory_points_%d' % b] = np.asarray(r['geo_memory_points'], np.float32)[::MEM_STRIDE]
        out['grm_geo_query_num_%d' % b] = np.int64(r['geo_query_num'])
        out['grm_sel_q_%d' % b] = np.concatenate(o['sel'][0])
        out['grm_sel_m_%d' % b] = o['sel'][1]
        pred = np.concatenate([np.zeros(3), bx[0, 3:6] * 1.05, [0.0]]).astype(np.float32)
        res = grm_mod.WaymoGeometryDataset.revert_to_each_frame({'pred_boxes': [pred], 'geo_trajectory': [r['geo_trajectory']],
                                                                 'pose': [info['pose']]})
        out['grm_pred_%d' % b], out['grm_revert_lidar_%d' % b] = pred, res[0].reshape(L, 7)
        print('track %d: L %d, points per box %d..%d' % (b, L, out['counts_%d' % b].min(), out['counts_%d' % b].max()))
    np.savez_compressed(os.path.join(HERE, 'refine_data.npz'), **out)


R_P2CO = ['xyz', 'intensity', 'p2co', 'score']
MEM_STRIDE = 8          # every 8th GRM memory row is stored

if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else '/root/reference')

"""Golden vectors for scoring the refiners against ground truth (tests/golden/refine_score.npz), produced by the reference's own
PositionRefineModel / GeometryRefineModel / ConfidenceRefineModel.generate_recall_record and daemon/generate_iou_gt.py's
generate_refine_boxes_iou on the CPU, class by class as refining/tools/test.py runs them.  The 3-D IoU the reference takes from the
compiled iou3d_nms op is served by the oracle's C restatement and .cuda() is the identity, as in make_golden_track_gt.py.  The
tracks are labelled by the reference's target_assign.assign_track_target; its result is regrouped per object (the host loop of
daemon/prepare_object_data.py:64-190, which needs the raw frame files) by oracle.refine_score_ref.attach_targets, and the PRM
inputs (pos_trajectory, gt_pos_trajectory) are the float32 roundings of the oracle's float64 init-box transform.

The scene (200 frames, world offsets of kilometres, the ego turning through +-pi):
  1  Vehicle, 200 boxes on a moving vehicle (dynamic): every other input box is 0.9 m off (under 0.7), the PRM lifts those over 0.7
     and drops every seventh box under it
  2  Vehicle, 25 boxes on a parked vehicle (static) that is labelled in the first 20 frames only
  3  Pedestrian, 10 boxes, 7 of them over 0.5 on the input side: a match ratio exactly on the 0.7 cut (>= for the PRM, > for the GRM)
  4  Cyclist, 10 boxes (dynamic)
  5  Vehicle, 1 box
  6  Vehicle, 10 boxes far from every object (unmatched)
  7  Pedestrian, 4 boxes, unmatched

    python tests/golden/make_golden_refine_score.py /path/to/reference
"""
import os
import pickle
import sys
import tempfile
from collections import defaultdict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

CLASS_NAMES = ('Vehicle', 'Pedestrian', 'Cyclist')
THRESHOLDS = {'Vehicle': [0.7, 0.5], 'Pedestrian': [0.5], 'Cyclist': [0.5]}
F, L = 200, 200
DIMS = {'Vehicle': [4.6, 2.0, 1.6], 'Pedestrian': [0.9, 0.9, 1.8], 'Cyclist': [1.9, 0.8, 1.7]}


def poses():
    P = np.zeros((F, 4, 4))
    for f in range(F):
        yaw = np.pi - 0.3 + 0.004 * f
        c, s = np.cos(yaw), np.sin(yaw)
        P[f, :3, :3] = [[c, -s, 0], [s, c, 0], [0, 0, 1]]
        P[f, :3, 3] = [5000.0 + 0.5 * f, -3000.0 + 0.1 * f, 50.0]
        P[f, 3, 3] = 1
    return P


def scene():
    """-> frames (info dicts), tracks {id: {'boxes_global', 'name', 'score', 'sample_idx', 'state'}}"""
    P = poses()
    objs = {
        'veh_a': ('Vehicle', range(0, 200), lambda f: [5010.0 + 0.3 * f, -2990.0, 49.0], 0.0),
        'veh_b': ('Vehicle', range(0, 20), lambda f: [4980.0, -3020.0, 49.0], 1.2),
        'ped_c': ('Pedestrian', range(0, 10), lambda f: [5020.0, -3010.0, 49.2], 0.0),
        'cyc_d': ('Cyclist', range(5, 15), lambda f: [5030.0 - 0.4 * f, -3005.0, 49.1], 3.1),
        'veh_e': ('Vehicle', range(50, 51), lambda f: [4960.0, -3040.0, 49.0], -2.9),
    }
    rows = [[] for _ in range(F)]
    world = {}
    for oid, (name, frs, cen, h) in objs.items():
        for f in frs:
            w = np.array(cen(f) + DIMS[name] + [h, 0.0, 0.0])
            world[(oid, f)] = w
            rows[f].append((name, oid, w))
    frames = []
    for f in range(F):
        R, t = P[f, :3, :3], P[f, :3, 3]
        yaw = np.arctan2(R[1, 0], R[0, 0])
        lid = [np.r_[(w[:3] - t) @ R, w[3:6], np.arctan2(np.sin(w[6] - yaw), np.cos(w[6] - yaw))] for _, _, w in rows[f]]
        n = len(rows[f])
        frames.append({'sequence_name': 'seq', 'sample_idx': f, 'frame_id': f, 'pose': P[f].copy(),
                       'annos': {'name': np.array([r[0] for r in rows[f]], dtype='<U10'),
                                 'obj_ids': np.array([r[1] for r in rows[f]], dtype='<U16'),
                                 'gt_boxes_lidar': np.array(lid, np.float32).reshape(-1, 7),
                                 'gt_boxes_global': np.array([r[2] for r in rows[f]], np.float64).reshape(-1, 9),
                                 'difficulty': np.zeros(n, np.int32), 'num_points_in_gt': np.full(n, 100, np.int32)}})
    far = np.array([5200.0, -2800.0, 49.0] + DIMS['Vehicle'] + [0.4, 0.0, 0.0])
    farp = np.array([5100.0, -3100.0, 49.2] + DIMS['Pedestrian'] + [0.0, 0.0, 0.0])
    # id -> (class, [(frame, world box)])
    tks = {
        1: ('Vehicle', [(f, world[('veh_a', f)] + np.r_[0.25 if f % 2 else 0.9, 0, 0, np.zeros(6)]) for f in range(200)]),
        2: ('Vehicle', [(f, world[('veh_b', min(f, 19))] + np.r_[0.1, 0.05, 0, np.zeros(6)]) for f in range(25)]),
        3: ('Pedestrian', [(f, world[('ped_c', f)] + np.r_[0.45 if f in (1, 4, 8) else 0.05, 0, 0, np.zeros(6)]) for f in range(10)]),
        4: ('Cyclist', [(f, world[('cyc_d', f)] + np.r_[0.1, 0.05, 0.02, np.zeros(6)]) for f in range(5, 15)]),
        5: ('Vehicle', [(50, world[('veh_e', 50)] + np.r_[0.2, 0, 0, np.zeros(3), 0.03, 0, 0])]),
        6: ('Vehicle', [(f, far) for f in range(30, 40)]),
        7: ('Pedestrian', [(f, farp) for f in range(100, 104)]),
    }
    tracks = {}
    for tid, (name, ents) in tks.items():
        t = defaultdict(list)
        n = len(ents)
        t.update({'boxes_global': np.array([w for _, w in ents]), 'name': np.array([name] * n),
                  'score': (0.3 + 0.6 * ((np.arange(n) * 7 + tid) % 10) / 10).astype(np.float32),
                  'sample_idx': np.array([str(f) for f, _ in ents]), 'obj_ids': np.full(n, tid),
                  'state': 'dynamic' if tid in (6,) else 'static'})
        tracks[tid] = t
    return frames, tracks


def predictions(infos):
    """-> PRM boxes in the init-box frame (B, L, 7) f32, GRM boxes (B, 7) f32, CRM scores (B, L) f32, seeded"""
    from oracle import refine_score_ref as R
    g = np.random.default_rng(11)
    B = len(infos)
    prm, grm, crm = np.zeros((B, L, 7), np.float32), np.zeros((B, 7), np.float32), np.zeros((B, L), np.float32)
    for b, (tid, info) in enumerate(infos.items()):
        n = len(info['boxes_global'])
        tgt = np.where(info['matched'][:, None] & info['matched_tracklet'], info['gt_boxes_global'], info['boxes_global'])
        tgt = tgt + np.r_[0.04, -0.03, 0.01, 0.02, 0.01, 0.0, 0.01]
        if tid == 1:
            tgt[::7, 0] += 1.2
        prm[b, :n] = R.init_frame_boxes(tgt, info['boxes_global'][n // 2])
        size = tgt[0, 3:6] * (1.6 if tid == 2 else 1.03)
        grm[b] = np.r_[g.normal(0, 0.1, 3), size, 0.0]
        crm[b, :n] = g.uniform(0.05, 0.95, n)
    return prm, grm, crm


def revert(prm, info):
    """box_coords_transform: PRM boxes back to the world, float64"""
    from oracle import refine_score_ref as R
    n = len(info['boxes_global'])
    return R.world_boxes(prm[:n], info['boxes_global'][n // 2])


def pack(rec):
    keys = [k for k in rec if not isinstance(rec[k], list)]
    return np.array(keys), np.array([int(rec[k]) for k in keys], np.int64)


def main():
    import make_golden_track_gt as mg
    mg.install()
    import ref_import
    ref_import._pkg('daemon', ref_import.REF + '/daemon')
    sys.modules['detzero_utils.common_utils'] = type(sys)('detzero_utils.common_utils')
    sys.modules['detzero_utils.common_utils'].create_logger = lambda *a, **k: None
    sys.modules['detzero_utils'].common_utils = sys.modules['detzero_utils.common_utils']
    from daemon.generate_iou_gt import generate_refine_boxes_iou
    from detzero_b200.config import AttrDict
    from detzero_refine.models.confidence_refine_model import ConfidenceRefineModel
    from detzero_refine.models.geometry_refine_model import GeometryRefineModel
    from detzero_refine.models.position_refine_model import PositionRefineModel
    from detzero_track.models.tracking_modules import target_assign
    from oracle import refine_score_ref as R

    frames, tracks = scene()
    gt = {str(fr['sample_idx']): fr for fr in frames}
    assigned = target_assign.assign_track_target((gt, mg.fresh(tracks), gt), {'Vehicle': 0.3, 'Pedestrian': 0.1, 'Cyclist': 0.1})
    infos_all = R.attach_targets(assigned)
    infos_all = {tid: infos_all[tid] for tid in tracks}                      # track id order
    prm, grm, crm = predictions(infos_all)
    out = {}
    out['gt_counts'] = np.array([len(fr['annos']['name']) for fr in frames], np.int32)
    for k in ('name', 'obj_ids', 'gt_boxes_lidar', 'gt_boxes_global', 'difficulty', 'num_points_in_gt'):
        out['gt_' + k] = np.concatenate([fr['annos'][k] for fr in frames])
    out['poses'] = np.stack([fr['pose'] for fr in frames])
    ids = list(tracks)
    out['tk_ids'] = np.array(ids, np.int64)
    out['tk_counts'] = np.array([len(tracks[t]['name']) for t in ids], np.int32)
    out['tk_boxes'] = np.concatenate([tracks[t]['boxes_global'] for t in ids])
    out['tk_name'] = np.concatenate([tracks[t]['name'] for t in ids])
    out['tk_frame'] = np.concatenate([tracks[t]['sample_idx'].astype(np.int32) for t in ids])
    out['tk_score'] = np.concatenate([tracks[t]['score'] for t in ids])
    out['tk_dynamic'] = np.array([tracks[t]['state'] == 'dynamic' for t in ids])
    out['label_tk'] = np.array(list(assigned['label']), np.int64)
    out['label_obj'] = np.array([assigned['label'][t]['gt']['obj_ids'][0] for t in assigned['label']], dtype='<U16')
    out['label_state'] = np.array([assigned['label'][t]['track']['state'] == 'dynamic' for t in assigned['label']])
    out['unlabel_tk'] = np.array(list(assigned['unlabel']), np.int64)
    out['prm_pred'], out['grm_pred'], out['crm_pred'] = prm, grm, crm
    labels = {}
    for c in CLASS_NAMES:
        th = THRESHOLDS[c]
        sel = [b for b, t in enumerate(ids) if infos_all[t]['name'] == c]
        infos = [infos_all[ids[b]] for b in sel]
        n = [len(i['boxes_global']) for i in infos]
        pad = lambda a: np.concatenate([a, np.zeros((L - len(a), 7))]).astype(np.float32)
        base = {'box_num': n, 'state': [i['state'] for i in infos], 'matched': [i['matched'] for i in infos],
                'matched_tracklet': [i['matched_tracklet'] for i in infos]}
        d = dict(base)
        d['pos_init_box'] = torch.zeros(len(sel), 7)
        d['pos_trajectory'] = torch.from_numpy(np.stack([pad(R.init_frame_boxes(i['boxes_global'], i['boxes_global'][k // 2]))
                                                         for i, k in zip(infos, n)]))
        d['gt_pos_trajectory'] = torch.from_numpy(np.stack([pad(R.gt_pos_trajectory(i)) for i in infos]))
        rec = PositionRefineModel.generate_recall_record(torch.from_numpy(prm[sel]), {}, d, th)
        out['PRM_%s_keys' % c], out['PRM_%s_vals' % c] = pack(rec)
        d = dict(base)
        d['geo_trajectory'] = [i['boxes_global'].copy() for i in infos]
        d['gt_geo_trajectory'] = [i['gt_boxes_global'].copy() for i in infos]
        d['gt_geo_query_boxes'] = np.ones((len(sel), 3, 7))
        m = GeometryRefineModel.__new__(GeometryRefineModel)
        m.model_cfg = AttrDict({'POST_PROCESSING': AttrDict({'CENTER_ALIGN': False})})
        rec = GeometryRefineModel.generate_recall_record(m, torch.from_numpy(grm[sel]), {}, d, th)
        out['GRM_%s_keys' % c], out['GRM_%s_vals' % c] = pack(rec)
        # the CRM labels: generate_refine_boxes_iou on the PRM / GRM result pickles
        with tempfile.TemporaryDirectory() as tmp:
            geo = {'seq': {ids[b]: {'boxes_lidar': np.tile(grm[b], (k, 1))} for b, k in zip(sel, n)}}
            pos = {'seq': {ids[b]: {'boxes_global': revert(prm[b], i), 'boxes_gt_global': i['gt_boxes_global']}
                           for b, i in zip(sel, infos)}}
            gp, pp = os.path.join(tmp, 'geo_train.pkl'), os.path.join(tmp, 'pos_train.pkl')
            pickle.dump(geo, open(gp, 'wb'))
            pickle.dump(pos, open(pp, 'wb'))
            generate_refine_boxes_iou(c, gp, pp, tmp, type('Log', (), {'info': staticmethod(lambda *a: None)})())
            iou = pickle.load(open(os.path.join(tmp, '%s_iou_train.pkl' % c), 'rb'))['seq']
        labels.update(iou)
        pad1 = lambda a: np.concatenate([np.asarray(a, np.float32), np.full(L - len(a), -1, np.float32)])
        d = {'batch_size': len(sel), 'box_num': n, 'state': base['state'], 'matched_tracklet': base['matched_tracklet'],
             'conf_score': torch.from_numpy(np.stack([pad1(i['score']) for i in infos])) if sel else torch.zeros(0, L),
             'pred_score': torch.from_numpy(crm[sel]), 'iou': torch.from_numpy(np.stack([pad1(iou[ids[b]]) for b in sel]))}
        rec = ConfidenceRefineModel.generate_recall_record(None, {}, d, th)
        out['CRM_%s_keys' % c], out['CRM_%s_vals' % c] = pack(rec)
        out['CRM_%s_all_keys' % c] = np.array(list(rec))
        for k in ('gt_score', 'pred_score', 'ori_score'):
            out['CRM_%s_%s' % (c, k)] = np.array(rec[k])
        print(c, {k: int(v) for k, v in zip(*pack(rec))})
        print(c, 'PRM', dict(zip(out['PRM_%s_keys' % c].tolist(), out['PRM_%s_vals' % c].tolist())))
        print(c, 'GRM', dict(zip(out['GRM_%s_keys' % c].tolist(), out['GRM_%s_vals' % c].tolist())))
    out['refine_iou'] = np.concatenate([np.asarray(labels[t], np.float32) for t in ids])
    path = os.path.join(HERE, 'refine_score.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes): labels %s, unlabelled %s' % (path, os.path.getsize(path), out['label_tk'].tolist(),
                                                           out['unlabel_tk'].tolist()))


if __name__ == '__main__':
    if len(sys.argv) > 1:
        import ref_import
        ref_import.REF = sys.argv[1]
    main()

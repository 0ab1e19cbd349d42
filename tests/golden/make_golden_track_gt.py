"""Golden vectors for scoring tracks against ground truth (tests/golden/track_gt.npz), produced by the reference's own
target_assign.assign_track_target (BEV, REFINING.IOU_THRESHOLDS of waymo_detzero_track.yaml), TrackRecall.eval_single_seq and
TrackRecall.calculate_tracklet_recall (3-D IoU, eval_track.py's defaults) on the CPU, with numpy >= 2.  The rotated BEV IoU / overlap
and the 3-D IoU the reference takes from the compiled iou3d_nms_cuda op are served by the oracle's C restatement; np.int is aliased
as in make_golden_track.py; the track dicts are defaultdict(list) as TrackManager emits them and the frame keys strings as
sequence_list_to_dict makes them.

The scene (12 frames, km world offsets, the ego turning through +-pi): a fragmented vehicle (two tracks, the longer one labelled), an
id switch (one track over two vehicles), a pedestrian and a pedestrian track that never share a frame, a Sign row on a tracked vehicle
(masked), a cyclist with one difficulty-2 box (matched: L2), unmatched objects bucketed by their first box, frame 10 with ground truth
and no track, frame 11 with a track and no ground truth, and a pedestrian whose 3-D IoU passes 0.5 in exactly 3 of its 10 frames (a
match rate on the 0.3 cutoff).

    python tests/golden/make_golden_track_gt.py /path/to/reference
"""
import os
import sys
from collections import defaultdict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

CLASS_NAMES = ('Vehicle', 'Pedestrian', 'Cyclist')
F = 12
DIMS = {'Vehicle': [4.6, 2.0, 1.6], 'Pedestrian': [0.9, 0.9, 1.8], 'Cyclist': [1.9, 0.8, 1.7], 'Sign': [0.5, 0.5, 0.8]}


def poses():
    P = np.zeros((F, 4, 4))
    for f in range(F):
        yaw = np.pi - 0.3 + 0.06 * f
        c, s = np.cos(yaw), np.sin(yaw)
        P[f, :3, :3] = [[c, -s, 0], [s, c, 0], [0, 0, 1]]
        P[f, :3, 3] = [5000.0 + 1.5 * f, -3000.0 + 0.4 * f, 50.0]
        P[f, 3, 3] = 1
    return P


def scene():
    """-> frames (the info dicts), tracks {id: {'boxes_global', 'name', 'score', 'sample_idx'}}"""
    P = poses()
    # objects: id -> (class, frames, world centre at frame f, heading, difficulty per frame, num_points per frame)
    objs = {
        'veh_a': ('Vehicle', range(0, 10), lambda f: [5010.0 + 0.8 * f, -2990.0, 49.0], 0.3, {}, {}),
        'veh_b': ('Vehicle', range(0, 10), lambda f: [4980.0, -3020.0 + 0.5 * f, 49.0], 1.2, {}, {6: 4}),
        'veh_c': ('Vehicle', range(0, 10), lambda f: [4990.0, -2975.0, 49.0], -2.9, {}, {}),
        'ped_d': ('Pedestrian', range(0, 5), lambda f: [5020.0, -3010.0 + 0.1 * f, 49.2], 0.0, {}, {}),
        'cyc_e': ('Cyclist', range(2, 11), lambda f: [5030.0 - 0.4 * f, -3005.0, 49.1], 3.1, {5: 2}, {}),
        'veh_f': ('Vehicle', range(3, 9), lambda f: [4960.0, -3040.0, 49.0], 0.7, {}, {3: 2}),
        'ped_h': ('Pedestrian', range(1, 6), lambda f: [5040.0, -2960.0, 49.2], 2.0, {}, {}),
        'ped_g': ('Pedestrian', range(0, 10), lambda f: [5000.0 + 0.05 * f, -3030.0, 49.2], -1.0, {}, {}),
    }
    rows = [[] for _ in range(F)]
    world = {}
    for oid, (name, frs, cen, h, diff, npts) in objs.items():
        for f in frs:
            w = np.array(cen(f) + DIMS[name] + [h, 0.5, -0.2])
            world[(oid, f)] = w
            rows[f].append((name, oid, w, diff.get(f, 0), npts.get(f, 100)))
    for f in (2, 3, 4):                                                      # a Sign on vehicle a, listed first
        rows[f].insert(0, ('Sign', 'sign_s', np.r_[world[('veh_a', f)][:3], DIMS['Sign'], 0.3, 0.0, 0.0], 0, 50))
    frames = []
    for f in range(F):
        R, t = P[f, :3, :3], P[f, :3, 3]
        lid = [np.r_[(w[:3] - t) @ R, w[3:6], np.arctan2(np.sin(w[6] - np.arctan2(R[1, 0], R[0, 0])),
                                                         np.cos(w[6] - np.arctan2(R[1, 0], R[0, 0])))] for _, _, w, _, _ in rows[f]]
        frames.append({'sequence_name': 'seq', 'sample_idx': f, 'frame_id': f, 'pose': P[f].copy(),
                       'annos': {'name': np.array([r[0] for r in rows[f]], dtype='<U10'),
                                 'obj_ids': np.array([r[1] for r in rows[f]], dtype='<U16'),
                                 'gt_boxes_lidar': np.array(lid, np.float32).reshape(-1, 7),
                                 'gt_boxes_global': np.array([r[2] for r in rows[f]], np.float64).reshape(-1, 9),
                                 'difficulty': np.array([r[3] for r in rows[f]], np.int32),
                                 'num_points_in_gt': np.array([r[4] for r in rows[f]], np.int32)}})
    # tracks: id -> [(object or None, frame, offset (dx, dy))]
    def follow(oid, frs, dx=0.0, dy=0.0):
        return [(oid, f, (dx, dy)) for f in frs]
    tks = {
        3: follow('veh_a', range(0, 4), 0.1),                               # fragmented: the shorter piece
        7: follow('veh_a', range(4, 10), 0.2),                              # the longer piece (labelled)
        8: follow('veh_b', range(0, 5), 0.05) + follow('veh_c', range(5, 10), 0.05),     # id switch
        11: follow('veh_c', range(0, 7), 0.1),
        12: follow('ped_d', range(0, 5), 0.03),
        14: [(None, f, (0.0, 0.0)) for f in range(6, 10)],                  # at ped_d's last place, after it is gone
        15: follow('cyc_e', range(2, 10), 0.1),
        18: follow('ped_g', range(0, 10)),                                  # 3 frames on the box, 7 frames 0.45 m off
        21: [(None, f, (0.0, 0.0)) for f in range(8, 12)],                  # a far false positive through frame 11
    }
    tracks = {}
    for tid, ents in tks.items():
        boxes, names, fr = [], [], []
        for oid, f, (dx, dy) in ents:
            if tid == 14:
                w, name = world[('ped_d', 4)].copy(), 'Pedestrian'
            elif tid == 21:
                w, name = np.array([5200.0, -2800.0, 49.0] + DIMS['Vehicle'] + [0.0, 0.0, 0.0]), 'Vehicle'
            else:
                w, name = world[(oid, f)].copy(), objs[oid][0]
            if tid == 18 and f not in (2, 5, 8):
                dx = 0.45
            w[0] += dx
            w[1] += dy
            boxes.append(w)
            names.append(name)
            fr.append(str(f))
        t = defaultdict(list)
        t.update({'boxes_global': np.array(boxes), 'name': np.array(names), 'score': np.full(len(fr), 0.8, np.float32),
                  'sample_idx': np.array(fr), 'obj_ids': np.full(len(fr), tid)})
        tracks[tid] = t
    return frames, tracks


def install():
    import make_golden_track
    make_golden_track.install()
    import oracle
    iu = sys.modules['detzero_utils.ops.iou3d_nms.iou3d_nms_utils']
    iu.boxes_iou3d_gpu = lambda a, b: torch.from_numpy(oracle.boxes_iou3d(a.numpy(), b.numpy()))


def fresh(tracks):
    out = {}
    for tid, t in tracks.items():
        d = defaultdict(list)
        d.update({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in t.items()})
        out[tid] = d
    return out


def main():
    install()
    from detzero_track.models.tracking_modules import target_assign
    from detzero_track.utils import track_recall
    frames, tracks = scene()
    gt = {str(fr['sample_idx']): fr for fr in frames}
    thr = {'Vehicle': 0.3, 'Pedestrian': 0.1, 'Cyclist': 0.1}
    assign = target_assign.assign_track_target((gt, fresh(tracks), gt), thr)
    ev = track_recall.TrackRecall.eval_single_seq({'gt': gt, 'pred': fresh(tracks)}, list(CLASS_NAMES), ['l1', 'l2'],
                                                  dict(zip(CLASS_NAMES, [0.7, 0.5, 0.5])), method='3d')
    rec = track_recall.TrackRecall.__new__(track_recall.TrackRecall)
    rec.difficultys, rec.class_names, rec.match_rate_list = ['l1', 'l2'], list(CLASS_NAMES), np.arange(0, 10) * 0.1
    table = rec.calculate_tracklet_recall({'seq': ev})
    out = {}
    # inputs
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
    # assign mode: labels in order, their object, per-box iou, state; unlabelled tracks in order
    lab = assign['label']
    out['label_tk'] = np.array(list(lab), np.int64)
    out['label_obj'] = np.array([lab[t]['gt']['obj_ids'][0] for t in lab], dtype='<U16')
    out['label_state'] = np.array([lab[t]['track']['state'] == 'dynamic' for t in lab])
    out['label_iou'] = np.concatenate([lab[t]['track']['iou'] for t in lab])
    out['label_gt_sample_idx'] = np.concatenate([lab[t]['gt']['sample_idx'] for t in lab])
    out['unlabel_tk'] = np.array(list(assign['unlabel']), np.int64)
    # tracklet recall table
    for d in ('l1', 'l2'):
        for c in CLASS_NAMES:
            for k in ('tp', 'fp', 'gt_nums', 'pred_nums', 'precisions', 'recalls'):
                out['recall_%s_%s_%s' % (d, c, k)] = np.array(table[d][c][k])
    path = os.path.join(HERE, 'track_gt.npz')
    np.savez_compressed(path, **out)
    print('wrote %s: labels %s, unlabelled %s' % (path, dict(zip(out['label_tk'].tolist(), out['label_obj'].tolist())),
                                                  out['unlabel_tk'].tolist()))
    for d in ('l1', 'l2'):
        for c in CLASS_NAMES:
            print(d, c, 'tp', table[d][c]['tp'], 'gt', table[d][c]['gt_nums'][0], 'pred', table[d][c]['pred_nums'][0])


if __name__ == '__main__':
    if len(sys.argv) > 1:
        import ref_import
        ref_import.REF = sys.argv[1]
    main()

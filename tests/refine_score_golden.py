"""tests/golden/refine_score.npz back in the reference's forms: the frame dicts of the ground truth, the track dict, the refiner
predictions and the reference's records."""
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'refine_score.npz')
CLASS_NAMES = ('Vehicle', 'Pedestrian', 'Cyclist')
THRESHOLDS = {'Vehicle': [0.7, 0.5], 'Pedestrian': [0.5], 'Cyclist': [0.5]}
ASSIGN_THR = {'Vehicle': 0.3, 'Pedestrian': 0.1, 'Cyclist': 0.1}


def load():
    """-> golden arrays, frames (info dicts), tracks {id: {'boxes_global', 'name', 'score', 'sample_idx', 'state'}}"""
    g = np.load(PATH)
    frames, o = [], 0
    for f, n in enumerate(g['gt_counts']):
        sl = slice(o, o + n)
        frames.append({'sequence_name': 'seq', 'sample_idx': f, 'frame_id': f, 'pose': g['poses'][f],
                       'annos': {k: g['gt_' + k][sl] for k in ('name', 'obj_ids', 'gt_boxes_lidar', 'gt_boxes_global', 'difficulty',
                                                                'num_points_in_gt')}})
        o += n
    tracks, o = {}, 0
    for tid, n, dyn in zip(g['tk_ids'], g['tk_counts'], g['tk_dynamic']):
        sl = slice(o, o + n)
        tracks[int(tid)] = {'boxes_global': g['tk_boxes'][sl], 'name': g['tk_name'][sl], 'score': g['tk_score'][sl],
                            'sample_idx': np.array([str(f) for f in g['tk_frame'][sl]]), 'state': 'dynamic' if dyn else 'static'}
        o += n
    return g, frames, tracks


def record(g, model, cls):
    """the reference's record of one model ('PRM', 'GRM', 'CRM') and class: its integer entries, in the reference's key order"""
    return dict(zip(g['%s_%s_keys' % (model, cls)].tolist(), g['%s_%s_vals' % (model, cls)].tolist()))


def class_rows(g, cls):
    """indices (into the track id order) of the tracks of one class"""
    first = np.concatenate([[0], np.cumsum(g['tk_counts'])[:-1]])
    return [b for b in range(len(g['tk_ids'])) if g['tk_name'][first[b]] == cls]


def labels(g):
    """the reference's IoU labels per track, in track id order"""
    return np.split(g['refine_iou'], np.cumsum(g['tk_counts'])[:-1])

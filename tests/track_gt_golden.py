"""tests/golden/track_gt.npz back in the reference's forms: the frame dicts of the ground truth and the track dict."""
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'track_gt.npz')
CLASS_NAMES = ('Vehicle', 'Pedestrian', 'Cyclist')


def load():
    """-> golden arrays, frames (info dicts), tracks {id: {'boxes_global', 'name', 'score', 'sample_idx'}}"""
    g = np.load(PATH)
    frames, o = [], 0
    for f, n in enumerate(g['gt_counts']):
        sl = slice(o, o + n)
        frames.append({'sequence_name': 'seq', 'sample_idx': f, 'frame_id': f, 'pose': g['poses'][f],
                       'annos': {k: g['gt_' + k][sl] for k in ('name', 'obj_ids', 'gt_boxes_lidar', 'gt_boxes_global', 'difficulty',
                                                                'num_points_in_gt')}})
        o += n
    tracks, o = {}, 0
    for tid, n in zip(g['tk_ids'], g['tk_counts']):
        sl = slice(o, o + n)
        tracks[int(tid)] = {'boxes_global': g['tk_boxes'][sl], 'name': g['tk_name'][sl], 'score': np.full(n, 0.8, np.float32),
                            'sample_idx': np.array([str(f) for f in g['tk_frame'][sl]])}
        o += n
    return g, frames, tracks


def recall_table(g):
    return {d: {c: {k: g['recall_%s_%s_%s' % (d, c, k)] for k in ('tp', 'fp', 'gt_nums', 'pred_nums', 'precisions', 'recalls')}
                for c in CLASS_NAMES} for d in ('l1', 'l2')}

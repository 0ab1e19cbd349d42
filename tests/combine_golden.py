"""Readers of tests/golden/combine.npz (written by tests/golden/make_golden_combine.py): the per-track tables and drop dicts of its two
sequences, and the reference's frame list of each option pair."""
import os

import numpy as np
import torch

from oracle import combine_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'combine.npz')
SEQS = ('seq_a', 'seq_b')
#: combine_conf_res, combine_drop
VARIANTS = {'c1d1': (True, True), 'c1d0': (True, False), 'c0d1': (False, True), 'c0d0': (False, False)}


def load():
    return dict(np.load(GOLDEN))


def tables(g, s, L=200):
    """sequence s: the tables of refine.data.combine_frames (numpy, tracker scores in 'scores', CRM scores in 'crm'), poses,
    frame_ids"""
    trk = g['s%d_trk' % s]
    B = len(trk)
    t = {'prm_lidar': np.zeros((B, L, 7)), 'grm_pred': g['s%d_grm' % s], 'scores': np.zeros((B, L), np.float32),
         'crm': np.zeros((B, L), np.float32), 'frame_of_box': np.zeros((B, L), np.int32), 'box_num': trk[:, 3].astype(np.int32),
         'cls': trk[:, 0].astype(np.int32), 'track_id': trk[:, 1], 'poses': g['s%d_poses' % s], 'frame_ids': g['s%d_frame_ids' % s]}
    o = 0
    for b, (c, tid, first, n) in enumerate(trk):
        t['prm_lidar'][b, :n] = g['s%d_prm' % s][o:o + n]
        t['scores'][b, :n] = g['s%d_score' % s][o:o + n]
        t['crm'][b, :n] = g['s%d_crm' % s][o:o + n]
        t['frame_of_box'][b, :n] = np.arange(first, first + n)
        o += n
    return t


def det_drop_from_rows(det, counts, kept, poses, name, frame_ids):
    """TrackResult.to_reference's det_drop of one sequence's gathered rows, keyed by str(frame id) as combine_det looks it up"""
    from detzero_b200.track import TrackResult
    F = len(counts)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))                                # noqa: E731
    res = TrackResult(t(det[None]), t(np.asarray(counts)[None]), t(poses[None]), t(np.array([F])),
                      torch.zeros((1, 0, 6), dtype=torch.int32), torch.zeros(1, dtype=torch.int32),
                      torch.zeros((1, 0, 9), dtype=torch.float64), torch.zeros((1, 0)), torch.zeros((1, 0), dtype=torch.int32),
                      torch.zeros((1, 0), dtype=torch.int32), t(np.asarray(kept)[None]))
    return res.to_reference([name], [[str(x) for x in frame_ids]])[1][name]


def det_drop(g, s):
    return det_drop_from_rows(g['s%d_det' % s], g['s%d_counts' % s], g['s%d_kept' % s], g['s%d_poses' % s], SEQS[s],
                              g['s%d_frame_ids' % s])


def expected(g, v):
    """the reference's frame list (both sequences) of option pair v, poses from the sequences' input poses"""
    p = {k: g['%s_%s' % (v, k)] for k in ('frame', 'obj', 'rows', 'name')}
    p['pose'] = np.array([g['s%d_poses' % s][int(np.flatnonzero(g['s%d_frame_ids' % s] == fid)[0])] for s, fid in p['frame'][:, :2]])
    return combine_ref.unpack_frames(p, list(SEQS))


def oracle_frames(g, v):
    conf, drop = VARIANTS[v]
    out = []
    for s, name in enumerate(SEQS):
        t = tables(g, s)
        out += combine_ref.frame_list(t['prm_lidar'], t['grm_pred'], t['crm'] if conf else t['scores'], t['frame_of_box'], t['box_num'],
                                      t['cls'], t['track_id'], t['poses'], name, t['frame_ids'], det_drop(g, s) if drop else None)
    return out

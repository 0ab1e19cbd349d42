"""numpy restatement of DetZero's combine stage (daemon/combine_output.py:27-41,44-99,102-167) for one sequence: the per-track tables
of refine.data.combine_frames become the per-track dicts combine_final builds, then convert_frame_format's frame list, then
combine_det's dropped rows from the tracker's det_drop.  Pure data movement: the device must agree exactly.

Deviations kept as the device keeps them: every class of the tables in one list (the reference accumulates per-class files), and a
frame with tracks but no det_drop entry gets no dropped row (the reference raises KeyError).

pack_frames / unpack_frames store a frame list in flat arrays (tests/golden/combine.npz)."""
from collections import defaultdict

import numpy as np

CLASS_NAMES = ('Vehicle', 'Pedestrian', 'Cyclist')
KEYS = ('sequence_name', 'frame_id', 'obj_ids', 'name', 'score', 'boxes_lidar', 'boxes_global', 'pose')


def frame_list(prm_lidar, grm_pred, scores, frame_of_box, box_num, cls, track_id, poses, sequence_name, frame_ids, det_drop=None):
    """tables as refine.data.combine_frames takes them (numpy), poses (F, 4, 4), frame_ids[f] the id of sequence frame f, det_drop
    one sequence's {str(frame id): {'boxes_lidar', 'score', 'name', ...}} (TrackResult.to_reference's form) or None"""
    track_data = {}
    for b in range(len(box_num)):
        n = int(box_num[b])
        tid = int(track_id[b])
        assert tid not in track_data, 'track ids must be unique'
        lid = np.array(prm_lidar[b, :n], np.float64)
        lid[:, 3:6] = np.float64(np.asarray(grm_pred[b], np.float32)[3:6])          # combine_final :126-129
        track_data[tid] = {'sequence_name': sequence_name, 'boxes_lidar': lid, 'score': np.asarray(scores[b, :n], np.float32),
                           'name': [CLASS_NAMES[int(cls[b]) - 1]] * n, 'pose': [poses[f] for f in frame_of_box[b, :n]],
                           'sample_idx': np.array([str(frame_ids[f]) for f in frame_of_box[b, :n]])}
    # convert_frame_format
    out = []
    order_map = defaultdict(list)
    for tk_id, tk in track_data.items():
        for i, sa in enumerate(tk['sample_idx']):
            order_map[sa].append([tk_id, i])
    for frm in order_map:
        m = np.stack(order_map[frm])
        obj_ids, orders = m[:, 0], m[:, 1]
        n = len(obj_ids)
        boxes_lidar = np.zeros((n, 7), np.float32)
        score = np.zeros(n, np.float32)
        name = np.full(n, 'none', dtype=object)
        for i, oid in enumerate(obj_ids):
            boxes_lidar[i] = track_data[oid]['boxes_lidar'][orders[i]]
            score[i] = track_data[oid]['score'][orders[i]]
            name[i] = track_data[oid]['name'][orders[i]]
        out.append({'sequence_name': sequence_name, 'frame_id': int(frm), 'obj_ids': obj_ids, 'name': name, 'score': score,
                    'boxes_lidar': boxes_lidar, 'boxes_global': np.zeros((n, 9), np.float32),
                    'pose': track_data[obj_ids[0]]['pose'][orders[0]]})
    # combine_det
    if det_drop is not None:
        for fr in out:
            d = det_drop.get(str(fr['frame_id']))
            if d is None:
                continue
            for k in ('boxes_lidar', 'name', 'score'):
                fr[k] = np.concatenate([fr[k], d[k]], axis=0)
    return out


def assert_frames_equal(got, want):
    """two frame lists are equal: frame order, keys and their order, dtypes and shapes, and every value bit for bit"""
    assert len(got) == len(want), (len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        assert list(g) == list(w), (i, list(g), list(w))
        for k in w:
            a, b = g[k], w[k]
            if isinstance(b, np.ndarray):
                assert isinstance(a, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape, (i, k, getattr(a, 'dtype', type(a)),
                                                                                                b.dtype, np.shape(a), b.shape)
                if b.dtype == object:
                    assert list(a) == list(b), (i, k)
                else:
                    assert a.tobytes() == b.tobytes(), (i, k, a, b)
            else:
                assert type(a) is type(b) and a == b, (i, k, a, b)


def pack_frames(frames, sequence_names):
    """a frame list -> flat arrays: frame (n, 4) int64 [sequence index, frame id, rows, track rows], obj (sum track rows) int64,
    rows (sum rows, 8) float32 [boxes_lidar, score], name (sum rows) int8 class index, pose (n, 4, 4)"""
    fr, obj, rows, name, pose = [], [], [], [], []
    for d in frames:
        n, t = len(d['score']), len(d['obj_ids'])
        fr.append([sequence_names.index(d['sequence_name']), d['frame_id'], n, t])
        obj.append(np.asarray(d['obj_ids'], np.int64))
        rows.append(np.concatenate([d['boxes_lidar'], d['score'][:, None]], 1))
        name.append(np.array([CLASS_NAMES.index(x) for x in d['name']], np.int8))
        pose.append(d['pose'])
    return {'frame': np.asarray(fr, np.int64).reshape(-1, 4), 'obj': np.concatenate(obj) if obj else np.zeros(0, np.int64),
            'rows': np.concatenate(rows).astype(np.float32) if rows else np.zeros((0, 8), np.float32),
            'name': np.concatenate(name) if name else np.zeros(0, np.int8), 'pose': np.asarray(pose, np.float64).reshape(-1, 4, 4)}


def unpack_frames(p, sequence_names):
    out = []
    r = o = 0
    for i, (s, fid, n, t) in enumerate(p['frame']):
        rows = p['rows'][r:r + n]
        out.append({'sequence_name': sequence_names[s], 'frame_id': int(fid), 'obj_ids': p['obj'][o:o + t].copy(),
                    'name': np.array([CLASS_NAMES[c] for c in p['name'][r:r + n]], dtype=object), 'score': rows[:, 7].copy(),
                    'boxes_lidar': rows[:, :7].copy(), 'boxes_global': np.zeros((t, 9), np.float32), 'pose': p['pose'][i].copy()})
        r, o = r + n, o + t
    return out

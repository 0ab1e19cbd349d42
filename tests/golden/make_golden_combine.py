"""Golden vectors for the combine stage (tests/golden/combine.npz), produced by the reference's own combine_final
(daemon/combine_output.py) on seeded per-class refiner pickles and a tracker drop pickle in the reference's formats, written to a
temporary root.  combine_final runs with frame_save=True for combine_conf_res on and off, with and without combine_drop_path, and
the last class's <class>_final_frame.pkl of each run is stored.

The scene: two sequences (200 and 30 frames), each with tracks of all three classes, of 1 to 200 boxes; the first track of
sequence 0 starts late, so the frames' first-appearance order is not their sorted order; frames shared by tracks of different
classes; a frame with only dropped detections (it gets no row); a frame whose drop entry is empty; dropped headings beyond +-pi.
Every frame with a track has a drop entry (combine_det raises KeyError otherwise).

    python tests/golden/make_golden_combine.py /path/to/reference
"""
import logging
import os
import pickle
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

CLASS_NAMES = ('Vehicle', 'Pedestrian', 'Cyclist')
SEQS = ('seq_a', 'seq_b')
FRAMES = (200, 30)
K = 3
VARIANTS = {'c1d1': (True, True), 'c1d0': (True, False), 'c0d1': (False, True), 'c0d0': (False, False)}
# per sequence, per class: (first frame, box count) of each track, in track-id order
TRACKS = ({'Vehicle': [(150, 31), (0, 200), (57, 1)], 'Pedestrian': [(10, 40), (60, 3)], 'Cyclist': [(100, 25), (5, 12)]},
          {'Vehicle': [(12, 10)], 'Pedestrian': [(3, 27), (20, 2)], 'Cyclist': [(29, 1), (8, 6)]})


def scene(seed=7):
    g = np.random.default_rng(seed)
    out = []
    tid = 0
    for s, F in enumerate(FRAMES):
        yaw = g.uniform(-np.pi, np.pi) + 0.01 * np.arange(F)
        poses = np.zeros((F, 4, 4))
        poses[:, 0, 0], poses[:, 0, 1], poses[:, 1, 0], poses[:, 1, 1] = np.cos(yaw), -np.sin(yaw), np.sin(yaw), np.cos(yaw)
        poses[:, 2, 2] = poses[:, 3, 3] = 1
        poses[:, :3, 3] = [5000.0, -3000.0, 50.0] + np.cumsum(g.normal(0, 1, (F, 3)), 0)
        frame_ids = 1000 * (s + 1) + 7 * np.arange(F) + 3
        tracks = []
        for ci, c in enumerate(CLASS_NAMES):
            for first, n in TRACKS[s][c]:
                tid += int(g.integers(1, 4))
                prm = np.concatenate([g.uniform(-80, 80, (n, 2)), g.uniform(-3, 1, (n, 1)), g.uniform(0.5, 5, (n, 3)),
                                      g.uniform(-4, 4, (n, 1))], 1)
                grm = np.concatenate([g.uniform(-80, 80, 3), g.uniform(0.5, 5, 3), g.uniform(-3, 3, 1)]).astype(np.float32)
                tracks.append({'cls': ci + 1, 'id': tid, 'frames': np.arange(first, first + n), 'prm': prm, 'grm': grm,
                               'score': g.uniform(0, 1, n).astype(np.float32), 'crm': g.uniform(0, 1, n).astype(np.float32)})
        counts = g.integers(1, K + 1, F).astype(np.int32)
        det = np.zeros((F, K, 9), np.float32)
        det[..., :2] = g.uniform(-80, 80, (F, K, 2))
        det[..., 2] = g.uniform(-3, 1, (F, K))
        det[..., 3:6] = g.uniform(0.5, 5, (F, K, 3))
        det[..., 6] = g.uniform(-8, 8, (F, K))
        det[..., 7] = g.uniform(0, 1, (F, K))
        det[..., 8] = g.integers(1, 4, (F, K))
        kept = g.random((F, K)) < 0.5
        if s == 1:
            counts[0] = 0                            # no detection and no track
            kept[1] = False                          # frame 1: only dropped detections, no track
            kept[4, :counts[4]] = True               # frame 4: an empty drop entry
        else:
            kept[90, :counts[90]] = True
        out.append({'poses': poses, 'frame_ids': frame_ids, 'tracks': tracks, 'det': det, 'counts': counts, 'kept': kept})
    return out


def det_drop(sc, name):
    """the tracker's drop dict of one sequence, keyed by str(frame id) as combine_det looks frames up (TrackResult.to_reference)"""
    from tests.combine_golden import det_drop_from_rows
    return det_drop_from_rows(sc['det'], sc['counts'], sc['kept'], sc['poses'], name, sc['frame_ids'])


def write_pickles(root, scenes):
    res = os.path.join(root, 'result')
    os.makedirs(res)
    for c in CLASS_NAMES:
        pos, geo, conf = {}, {}, {}
        for name, sc in zip(SEQS, scenes):
            pos[name], geo[name], conf[name] = {}, {}, {}
            for tk in sc['tracks']:
                if CLASS_NAMES[tk['cls'] - 1] != c:
                    continue
                fr = [int(sc['frame_ids'][f]) for f in tk['frames']]
                n = len(fr)
                pose = [sc['poses'][f].copy() for f in tk['frames']]
                geo_lidar = [np.concatenate([tk['prm'][j, :3] + 0.1, np.float64(tk['grm'][3:6]), tk['prm'][j, 6:] - 0.1])[None]
                             for j in range(n)]                          # waymo_geometry_dataset.py: (1, 7) rows, the GRM size
                pos[name][tk['id']] = {'sequence_name': name, 'frame_id': fr, 'boxes_lidar': [tk['prm'][j].copy() for j in range(n)],
                                       'boxes_global': [np.zeros(7) for _ in range(n)], 'score': list(tk['score']),
                                       'name': [c] * n, 'state': 'dynamic', 'pose': pose, 'boxes_gt': [], 'boxes_gt_global': []}
                geo[name][tk['id']] = {'sequence_name': name, 'frame_id': fr, 'boxes_lidar': geo_lidar, 'score': list(tk['score']),
                                       'name': [c] * n, 'pose': pose}
                conf[name][tk['id']] = {'sequence_name': name, 'frame_id': np.asarray(fr), 'score': tk['score'].copy(),
                                        'new_score': tk['crm'].copy()}
        for kind, d in (('position', pos), ('geometry', geo), ('confidence', conf)):
            with open(os.path.join(res, '%s_%s_val.pkl' % (c, kind)), 'wb') as f:
                pickle.dump(d, f)
    drop_path = os.path.join(root, 'drop.pkl')
    with open(drop_path, 'wb') as f:
        pickle.dump({name: det_drop(sc, name) for name, sc in zip(SEQS, scenes)}, f)
    return drop_path


def install():
    import ref_import
    REF = ref_import.REF
    for name, path in (('detzero_utils', '/utils/detzero_utils'), ('detzero_track', '/tracking/detzero_track'),
                       ('detzero_track.utils', '/tracking/detzero_track/utils')):
        ref_import._pkg(name, REF + path)
    cu = types.ModuleType('detzero_utils.common_utils')                # only create_logger is imported; its module pulls in torch.distributed
    cu.create_logger = lambda *a, **k: logging.getLogger('combine')
    sys.modules['detzero_utils.common_utils'] = cu
    sys.path.insert(0, REF + '/daemon')
    import combine_output
    return combine_output


def main():
    co = install()
    scenes = scene()
    arrays = {}
    with tempfile.TemporaryDirectory() as root:
        drop_path = write_pickles(root, scenes)
        for v, (conf, drop) in VARIANTS.items():
            co.combine_final(root, list(CLASS_NAMES), logging.getLogger('combine'), split='val', combine_conf_res=conf,
                             combine_drop_path=drop_path if drop else None, track_save=False, frame_save=True)
            with open(os.path.join(root, 'result', '%s_final_frame.pkl' % CLASS_NAMES[-1]), 'rb') as f:
                frames = pickle.load(f)
            from oracle import combine_ref
            p = combine_ref.pack_frames(frames, list(SEQS))
            combine_ref.assert_frames_equal(combine_ref.unpack_frames(p, list(SEQS)), frames)     # the packing loses nothing
            for i, (s, fid) in enumerate(p['frame'][:, :2]):             # every pose is its frame's input pose: not stored again
                f = int(np.flatnonzero(scenes[s]['frame_ids'] == fid)[0])
                assert p['pose'][i].tobytes() == scenes[s]['poses'][f].tobytes()
            del p['pose']
            arrays.update({'%s_%s' % (v, k): a for k, a in p.items()})
    for s, sc in enumerate(scenes):
        tk = sc['tracks']
        arrays.update({'s%d_poses' % s: sc['poses'], 's%d_frame_ids' % s: sc['frame_ids'], 's%d_det' % s: sc['det'],
                       's%d_counts' % s: sc['counts'], 's%d_kept' % s: sc['kept'],
                       's%d_trk' % s: np.array([[t['cls'], t['id'], t['frames'][0], len(t['frames'])] for t in tk], np.int64),
                       's%d_prm' % s: np.concatenate([t['prm'] for t in tk]), 's%d_grm' % s: np.stack([t['grm'] for t in tk]),
                       's%d_score' % s: np.concatenate([t['score'] for t in tk]), 's%d_crm' % s: np.concatenate([t['crm'] for t in tk])})
    out = os.path.join(HERE, 'combine.npz')
    np.savez_compressed(out, **arrays)
    print('wrote %s: %d bytes, %s' % (out, os.path.getsize(out), {v: len(arrays[v + '_frame']) for v in VARIANTS}))


if __name__ == '__main__':
    if len(sys.argv) > 1:
        import ref_import
        ref_import.REF = sys.argv[1]
    main()

"""Golden vectors for the tracker (tests/golden/track.npz), produced by the reference's own DataProcessor, TrackManager and
PostProcessor on the CPU, configured by the shipped tracking/tools/cfgs/tk_model_cfgs/waymo_detzero_track.yaml and
tk_dataset_cfgs/waymo_dataset.yaml.  The rotated BEV IoU / overlap the reference takes from the compiled iou3d_nms_cuda op are served
by the oracle's C restatement.

The scene is detzero_b200.synthetic.synthetic_detections (lanes of parked, slow and fast vehicles, pedestrians and cyclists, misses,
low-score stretches, far false positives, a chain of static pedestrians forming one large association component), plus a frame with
no detections after the first, an overlap-filter score tie (a duplicate detection with an equal score), two weaker duplicates the
filter drops, and two nested vehicles born in the same frame, the smaller first, whose tracks merge.

    python tests/golden/make_golden_track.py /path/to/reference
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

CLASS_NAMES = ('Vehicle', 'Pedestrian', 'Cyclist')
SEED, FRAMES = 3, 40


def scene():
    from detzero_b200 import synthetic
    d = synthetic.synthetic_detections(SEED, frames=FRAMES, objects=40, false_positives=8, chain=6)
    boxes, counts = d['boxes'], d['counts']
    counts[25] = 0                                                           # an empty frame after the first
    n = counts[5]                                                            # score tie: a duplicate row, 2 cm away
    boxes[5, n] = boxes[5, 0]
    boxes[5, n, 0] += 0.02
    counts[5] += 1
    for f in (8, 30):                                                        # plain drops: a weaker copy 5 cm away
        n = counts[f]
        boxes[f, n] = boxes[f, 1]
        boxes[f, n, 1] += 0.05
        boxes[f, n, 7] *= 0.8
        counts[f] += 1
    R, t = d['poses'][:, :3, :3], d['poses'][:, :3, 3]
    for f in range(10, 20):                                                  # nested vehicles, the small one first
        w = np.array([5000.0 - 40.0 + 10.0 * 0.1 * f, -3000.0 - 120.0, 49.0])
        lid = (w - t[f]) @ R[f]
        yaw = np.arctan2(R[f][1, 0], R[f][0, 0])
        k = counts[f]
        rows = [[*lid, 3.0, 1.6, 1.5, -yaw, 0.9, 1], [*lid, 8.0, 2.6, 3.0, -yaw, 0.7, 1]]
        if f > 10:
            rows = rows[1:]
        for r in rows:
            boxes[f, k] = r
            k += 1
        counts[f] = k
    return boxes, counts, d['poses']


def install():
    import ref_import
    ref_import.install()
    import oracle
    REF = ref_import.REF
    np.int = int                                                             # removed in numpy 2; the reference still uses it
    fp = types.ModuleType('filterpy')
    fpk = types.ModuleType('filterpy.kalman')
    fpk.KalmanFilter = object                                                # AB3DMOT only, not in the shipped config
    sys.modules['filterpy'], sys.modules['filterpy.kalman'] = fp, fpk
    for name, sub in (('detzero_track', ''), ('detzero_track.models', '/models'), ('detzero_track.datasets', '/datasets'),
                      ('detzero_track.utils', '/utils')):
        ref_import._pkg(name, REF + '/tracking/detzero_track' + sub)
    sys.modules['detzero_utils.ops.roiaware_pool3d.roiaware_pool3d_utils'] = types.ModuleType('roiaware_pool3d_utils')
    iu = types.ModuleType('detzero_utils.ops.iou3d_nms.iou3d_nms_utils')
    iu.boxes_iou3d_gpu = iu.boxes_giou3d_gpu = None
    sys.modules['detzero_utils.ops.iou3d_nms.iou3d_nms_utils'] = iu
    cuda = sys.modules['detzero_utils.ops.iou3d_nms.iou3d_nms_cuda']

    def iou(a, b, out):
        out[...] = torch.from_numpy(oracle.boxes_iou_bev(a.numpy(), b.numpy()))

    def overlap(a, b, out):
        out[...] = torch.from_numpy(oracle.boxes_overlap_bev(a.numpy(), b.numpy()))
    cuda.boxes_iou_bev_gpu, cuda.boxes_overlap_bev_gpu = iou, overlap


def run_reference(boxes, counts, poses):
    import yaml
    from detzero_b200.config import AttrDict
    from detzero_track.datasets.data_processor import DataProcessor
    from detzero_track.models.tracking_modules import PostProcessor, TrackManager
    import ref_import
    cfg_dir = ref_import.REF + '/tracking/tools/cfgs/'
    with open(cfg_dir + 'tk_model_cfgs/waymo_detzero_track.yaml') as f:
        model = AttrDict(yaml.safe_load(f)['MODEL'])
    with open(cfg_dir + 'tk_dataset_cfgs/waymo_dataset.yaml') as f:
        data = AttrDict(yaml.safe_load(f))
    dets = {}
    for fr in range(len(counts)):
        n = int(counts[fr])
        dets[fr] = {'boxes_lidar': boxes[fr, :n, :7].copy(), 'score': boxes[fr, :n, 7].copy(),
                    'name': np.array([CLASS_NAMES[int(c) - 1] for c in boxes[fr, :n, 8]]), 'pose': poses[fr].copy(),
                    'frame_id': fr, 'sequence_name': 'seq'}
    processed, drop = DataProcessor(data.DATA_PROCESSOR).forward(dets)
    tracks = TrackManager(model.TRACKING).forward(processed)
    return PostProcessor(model.POST_PROCESS).forward(tracks), drop


def main():
    install()
    boxes, counts, poses = scene()
    tracks, drop = run_reference(boxes, counts, poses)
    kept = np.ones(boxes.shape[:2], bool)
    for fr, dd in drop.items():                                              # dropped rows, matched back by their exact values
        for b in dd['boxes_lidar']:
            i = np.flatnonzero((boxes[fr, :counts[fr], :6] == b[:6]).all(1))
            assert len(i) == 1
            kept[fr, i[0]] = False
    ids = sorted(tracks)
    trk, eb, es, eh, ef = [], [], [], [], []
    for tid in ids:
        t = tracks[tid]
        n = len(t['hit'])
        off = sum(len(x) for x in eh)
        trk.append([tid, CLASS_NAMES.index(t['name'][0]) + 1, int(t['sample_idx'][0]), n, int(t['state'] == 'dynamic'), off])
        eb.append(np.asarray(t['boxes_global'], np.float64))
        es.append(np.asarray(t['score'], np.float32))
        eh.append(np.asarray(t['hit'], np.int32))
        ef.append(np.asarray(t['sample_idx'], np.int32))
        assert all(x == t['name'][0] for x in t['name'])
    out = os.path.join(HERE, 'track.npz')
    np.savez_compressed(out, boxes=boxes, counts=counts, poses=poses, kept=kept, trk=np.asarray(trk, np.int32).reshape(-1, 6),
                        ent_box=np.concatenate(eb), ent_score=np.concatenate(es), ent_hit=np.concatenate(eh),
                        ent_frame=np.concatenate(ef))
    print('wrote %s: %d tracks, %d entries, %d dropped detections' % (out, len(ids), sum(len(x) for x in eh), int((~kept).sum())))


if __name__ == '__main__':
    if len(sys.argv) > 1:
        import ref_import
        ref_import.REF = sys.argv[1]
    main()

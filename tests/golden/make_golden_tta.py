"""Golden vectors for CenterPoint test-time augmentation (tests/golden/tta.npz), produced by the reference's own code on the CPU:
  * TestTimeAugmentor.forward (detection/detzero_det/datasets/augmentor/test_time_augmentor.py) with the TEST_TIME_AUGMENTOR block
    of detection/tools/cfgs/det_dataset_cfgs/waymo_1sweep.yaml, on a seeded ~1 K-point cloud with points outside the range;
  * CenterPoint.test_time_augment (detection/detzero_det/models/centerpoint.py:131-208) and, through it, wbf_online /
    weighted_boxes_fusion_3d (utils/ensemble_utils), on one frame of 15 seeded synthetic view detections.  The rotated BEV overlap
    that boxes_iou3d_gpu takes from the compiled iou3d_nms_cuda op is served by the oracle's C restatement.

    python tests/golden/make_golden_tta.py /path/to/reference
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)


def cloud():
    g = np.random.default_rng(11)
    n = 1024
    xy = g.uniform(-85.0, 85.0, (n, 2))                     # [-75.2, 75.2] is the range: ~20 % of the points lie outside
    z = g.uniform(-2.5, 4.5, (n, 1))
    return np.concatenate([xy, z, g.uniform(0, 1, (n, 2))], 1).astype(np.float32)


def _to_view(b, op, p):
    """an original-frame box as a detector would see it in view `op` (the inverse of the un-augmentation, up to rounding)"""
    b = b.copy()
    if op == 'flip_x':
        b[:, 1] = -b[:, 1]; b[:, 6] = -b[:, 6]
    elif op == 'flip_y':
        b[:, 0] = -b[:, 0]; b[:, 6] = -b[:, 6] - np.pi
    elif op == 'flip_xy':
        b[:, 0:2] = -b[:, 0:2]; b[:, 6] = b[:, 6] + np.pi
    elif op == 'rot':
        c, s = np.cos(p), np.sin(p)
        b[:, 0], b[:, 1] = b[:, 0] * c - b[:, 1] * s, b[:, 0] * s + b[:, 1] * c
        b[:, 6] = b[:, 6] + p
    elif op == 'scale':
        b[:, :6] *= p
    return b


def view_detections(names):
    """one frame of V view detections: ~150 objects, each seen by most views with per-view jitter, 3 labels, distinct scores"""
    from oracle import tta_ref
    g = np.random.default_rng(5)
    n_obj = 150
    lab = g.integers(1, 4, n_obj)
    size = np.array([[4.5, 2.0, 1.6], [0.9, 0.9, 1.8], [1.8, 0.7, 1.7]])[lab - 1] * g.uniform(0.85, 1.15, (n_obj, 3))
    xy = g.uniform(-60, 60, (n_obj, 2))
    xy[100:120] = xy[80:100] + g.normal(0, 0.8, (20, 2))     # near neighbours: clusters that compete
    obj = np.concatenate([xy, g.uniform(-0.5, 1.0, (n_obj, 1)), size, g.uniform(-np.pi, np.pi, (n_obj, 1))], 1)
    base = g.uniform(0.02, 0.95, n_obj)
    per_view = []
    for op, p in tta_ref.view_ops(names):
        keep = g.random(n_obj) < 0.9
        b = obj[keep] + np.concatenate([g.normal(0, 0.08, (keep.sum(), 3)), g.normal(0, 0.05, (keep.sum(), 3)),
                                        g.normal(0, 0.03, (keep.sum(), 1))], 1)
        b = _to_view(b, op, p).astype(np.float32)
        s = (np.clip(base[keep] + g.normal(0, 0.05, keep.sum()), 0.005, 0.99) + g.uniform(0, 1e-3, keep.sum())).astype(np.float32)
        o = np.argsort(-s, kind='stable')
        per_view.append((b[o], s[o], lab[keep][o]))
    scores = np.concatenate([s for _, s, _ in per_view])
    assert np.unique(scores).size == scores.size, 'score tie'
    return per_view


def main(ref):
    import ref_import
    ref_import.REF = ref
    ref_import.install()
    import oracle
    iou_mod = sys.modules['detzero_utils.ops.iou3d_nms.iou3d_nms_cuda']

    def boxes_overlap_bev_gpu(a, b, out):
        out.copy_(torch.from_numpy(oracle.boxes_overlap_bev(a.numpy(), b.numpy())))
    iou_mod.boxes_overlap_bev_gpu = boxes_overlap_bev_gpu
    torch.cuda.FloatTensor = lambda size: torch.zeros(size, dtype=torch.float32)      # boxes_iou3d_gpu's output buffer, on the CPU

    # the datasets package __init__ pulls in the spconv voxelizer: expose the augmentor directory only
    ref_import._pkg('detzero_det.datasets', ref + '/detection/detzero_det/datasets')
    ref_import._pkg('detzero_det.datasets.augmentor', ref + '/detection/detzero_det/datasets/augmentor')
    import yaml
    from detzero_b200.config import AttrDict
    from detzero_det.datasets.augmentor.test_time_augmentor import TestTimeAugmentor
    from detzero_det.models import centerpoint as ref_cp
    with open(os.path.join(ref, 'detection/tools/cfgs/det_dataset_cfgs/waymo_1sweep.yaml')) as f:
        cfg = AttrDict(yaml.safe_load(f))

    pts = cloud()
    views = TestTimeAugmentor(cfg.TEST_TIME_AUGMENTOR).forward({'points': pts.copy()})
    names = list(views.keys())
    aug = np.stack([views[n]['points'].astype(np.float32) for n in names])

    per_view = view_detections(names)
    pred_dicts = [{'pred_boxes': torch.from_numpy(b), 'pred_scores': torch.from_numpy(s), 'pred_labels': torch.from_numpy(l)}
                  for b, s, l in per_view]
    seen = {}
    real_wbf = ref_cp.wbf_online

    def spy(boxes, scores, labels):
        seen.update(boxes=boxes.clone().numpy(), scores=scores.clone().numpy(), labels=labels.clone().numpy())
        return real_wbf(boxes, scores, labels)
    ref_cp.wbf_online = spy
    fb, fs, fl = ref_cp.CenterPoint.test_time_augment({'tta_ops': names, 'batch_size': len(names)}, pred_dicts)
    K = max(len(b) for b, _, _ in per_view)
    raw = np.zeros((len(names), K, 7), np.float32)
    raw_s = np.zeros((len(names), K), np.float32)
    raw_l = np.zeros((len(names), K), np.int64)
    for v, (b, s, l) in enumerate(per_view):
        raw[v, :len(b)], raw_s[v, :len(b)], raw_l[v, :len(b)] = b, s, l
    np.savez_compressed(os.path.join(HERE, 'tta.npz'), names=np.array(names), points=pts, aug_points=aug,
                        view_boxes=raw, view_scores=raw_s, view_labels=raw_l,
                        unaug_boxes=seen['boxes'].astype(np.float32), fused_boxes=fb.numpy(), fused_scores=fs.numpy(),
                        fused_labels=fl.numpy().astype(np.int64))
    print('views %d, points %d, boxes in %d, fused %d' % (len(names), len(pts), int((raw_l > 0).sum()), len(fb)))


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else '/root/reference')

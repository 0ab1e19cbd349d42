"""CenterPoint test-time augmentation on the device (csrc/tta.cu, det/tta.py, CenterPoint TTA path) against the host
restatement oracle/tta_ref.py, which tests/test_tta_oracle.py pins to the reference's own outputs."""
import os

import numpy as np
import pytest
import torch

import oracle
from oracle import det_ref, tta_ref, weights
from tests import util

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'tta.npz')
NAMES = [str(n) for n in np.load(GOLD)['names']]


def _aug():
    from detzero_b200.det.tta import ops_from_names
    return ops_from_names(NAMES)


def _collate(frames):
    return np.concatenate([np.pad(p, ((0, 0), (1, 0)), constant_values=b) for b, p in enumerate(frames)]).astype(np.float32)


@pytest.mark.parametrize('c', [5, 6])
def test_expand_bit_exact(cuda, c):
    from detzero_b200 import ops
    frames = [util.config1_cloud(20000, 3, c=c), util.config1_cloud(7000, 4, c=c)]
    out = ops.tta_expand(torch.from_numpy(_collate(frames)).to(cuda), [len(f) for f in frames], _aug().expand_views()).cpu().numpy()
    V, row = len(NAMES), 0
    for b, f in enumerate(frames):
        for v, q in enumerate(tta_ref.augment(f, NAMES)):
            got = out[row:row + len(f)]
            assert np.all(got[:, 0] == b * V + v)
            assert np.array_equal(got[:, 1:].view(np.uint32), q.view(np.uint32)), (b, NAMES[v])
            row += len(f)
    assert row == out.shape[0]


def test_expand_then_voxelize_equals_masked_views(cuda):
    """the reference masks each augmented view to the x/y range before voxelizing; the device voxelizers alone give the same voxels"""
    from detzero_b200 import ops
    from detzero_b200.det.dataset import mask_points_by_range
    from detzero_b200.det.vfe import MeanVFE, DynamicMeanVFE
    rng = util.WAYMO_RANGE
    frame = util.config1_cloud(30000, 8, pc_range=[-80, -80, -2, 80, 80, 4], c=5)
    views = tta_ref.augment(frame, NAMES)
    masked = [q[mask_points_by_range(q, rng)] for q in views]
    assert sum(len(q) for q in masked) < len(frame) * len(NAMES)
    exp = ops.tta_expand(torch.from_numpy(_collate([frame])).to(cuda), [len(frame)], _aug().expand_views())
    V = len(NAMES)
    vfe = MeanVFE(None, 5, point_cloud_range=rng, voxel_size=util.VOXEL, max_num_voxels=200000)
    got = vfe({'points': exp, 'batch_size': V, 'points_per_frame': [len(frame)] * V})
    m = int(got['voxel_count'].item())
    ref = oracle.Point2VoxelCPU3d(util.VOXEL, rng, 5, 5, 200000)
    rv, rc, rn = [], [], []
    for v, q in enumerate(masked):
        a, cc, n = ref.point_to_voxel(q)
        rv.append(a); rn.append(n); rc.append(np.pad(cc, ((0, 0), (1, 0)), constant_values=v))
    rv, rc, rn = np.concatenate(rv), np.concatenate(rc), np.concatenate(rn)
    assert m == rv.shape[0]
    assert np.array_equal(got['voxel_coords'][:m].cpu().numpy(), rc)
    assert np.array_equal(got['voxel_num_points'][:m].cpu().numpy(), rn)
    assert np.array_equal(got['voxels'][:m].cpu().numpy().view(np.uint32), rv.view(np.uint32))
    vfe2 = MeanVFE(None, 5, point_cloud_range=rng, voxel_size=util.VOXEL, max_num_voxels=200000)
    plain = vfe2({'points': torch.from_numpy(_collate(masked)).to(cuda), 'batch_size': V, 'points_per_frame': [len(q) for q in masked]})
    assert torch.equal(got['voxel_features'][:m], plain['voxel_features'][:m])
    # DynamicMeanVFE on 6-column points
    frame6 = util.config1_cloud(20000, 9, pc_range=[-12, -12, -2, 12, 12, 4], c=6)
    views6 = tta_ref.augment(frame6, NAMES)
    masked6 = [q[mask_points_by_range(q, util.SMALL_RANGE)] for q in views6]
    exp6 = ops.tta_expand(torch.from_numpy(_collate([frame6])).to(cuda), [len(frame6)], _aug().expand_views())
    grid = [192, 192, 40]
    dyn = DynamicMeanVFE({}, 6, util.VOXEL, grid, util.SMALL_RANGE)
    d = dyn({'points': exp6, 'batch_size': V})
    md = int(d['voxel_count'].item())
    d2 = dyn({'points': torch.from_numpy(_collate(masked6)).to(cuda), 'batch_size': V})
    _, coords_ref = det_ref.dynamic_mean_vfe(_collate(masked6), util.SMALL_RANGE, util.VOXEL, grid)
    assert md == coords_ref.shape[0] == int(d2['voxel_count'].item())
    assert torch.equal(d['voxel_coords'][:md].cpu(), coords_ref)
    assert util.rel_err(d['voxel_features'][:md].cpu(), d2['voxel_features'][:md].cpu()) < 1e-5


def test_unaugment_within_2_ulp(cuda):
    from detzero_b200 import ops
    g = np.load(GOLD)
    V, K = g['view_boxes'].shape[:2]
    rows = np.concatenate([g['view_boxes'], g['view_scores'][..., None], g['view_labels'][..., None].astype(np.float32)], 2)
    counts = (g['view_labels'] > 0).sum(1).astype(np.int32)
    out = ops.tta_unaugment(torch.from_numpy(rows).to(cuda), torch.from_numpy(counts).to(cuda), _aug().unaugment_views()).cpu().numpy()
    ref = tta_ref.unaugment(g['view_boxes'], NAMES)
    for v in range(V):
        n = counts[v]
        ulp = np.spacing(np.abs(ref[v, :n]).astype(np.float32))
        assert np.all(np.abs(out[v, :n, :7] - ref[v, :n]) <= 2 * ulp), NAMES[v]
        assert np.array_equal(out[v, :n, 7:], rows[v, :n, 7:])
        assert np.all(out[v, n:] == 0)


def _wbf_check(got_boxes, got_n, ref):
    n = int(got_n)
    assert n == len(ref['scores'])
    g = got_boxes[:n]
    assert np.array_equal(g[:, 8].astype(np.int64), ref['labels'])
    assert np.all(np.abs(g[:, :7] - ref['boxes']) <= 1e-5 * np.maximum(np.abs(ref['boxes']), 1.0))
    assert np.all(np.abs(g[:, 7] - ref['scores']) <= 1e-6 * np.abs(ref['scores']))
    assert np.all(got_boxes[n:] == 0)


def _rows(boxes, scores, labels):
    return np.concatenate([boxes, scores[..., None], labels[..., None].astype(np.float32)], 2).astype(np.float32)


def _random_views(seed, V=15, K=500):
    g = np.random.default_rng(seed)
    n_obj = 420
    lab = g.integers(1, 4, n_obj)
    size = np.array([[4.5, 2.0, 1.6], [0.9, 0.9, 1.8], [1.8, 0.7, 1.7]])[lab - 1] * g.uniform(0.85, 1.15, (n_obj, 3))
    obj = np.concatenate([g.uniform(-70, 70, (n_obj, 2)), g.uniform(-0.5, 1, (n_obj, 1)), size, g.uniform(-np.pi, np.pi, (n_obj, 1))], 1)
    base = g.uniform(0.02, 0.95, n_obj)
    base[lab == 3] = g.uniform(0.0, 0.009, (lab == 3).sum())           # label 3: everything under its skip threshold
    boxes = np.zeros((V, K, 7), np.float32); scores = np.zeros((V, K), np.float32); labels = np.zeros((V, K), np.int64)
    counts = np.zeros(V, np.int32)
    for v in range(V):
        keep = np.nonzero(g.random(n_obj) < 0.9)[0]
        n = K if v % 3 == 0 else min(len(keep), K)                     # every third view full: padded with false positives
        pick = np.concatenate([keep, g.integers(0, n_obj, max(0, n - len(keep)))])[:n]
        b = obj[pick] + np.concatenate([g.normal(0, 0.1, (n, 3)), g.normal(0, 0.05, (n, 3)), g.normal(0, 0.03, (n, 1))], 1)
        boxes[v, :n], scores[v, :n], labels[v, :n] = b, base[pick] + g.uniform(0, 0.01, n) * (lab[pick] != 3), lab[pick]
        counts[v] = n
    return boxes, scores, labels, counts


def test_wbf_matches_oracle(cuda):
    from detzero_b200 import ops
    from detzero_b200.det import tta
    g = np.load(GOLD)
    V, K = g['view_boxes'].shape[:2]
    un = tta_ref.unaugment(g['view_boxes'], NAMES)
    counts = (g['view_labels'] > 0).sum(1).astype(np.int32)
    cases = [(un, g['view_scores'], g['view_labels'], counts)] + [_random_views(s) for s in (1, 2)]
    outs = []
    for boxes, scores, labels, cnt in cases:
        ref = tta_ref.wbf_3d(boxes, scores, labels)
        assert ref['min_margin'] > 1e-5
        assert any(len(m) > 1 for m in ref['members'])
        rows = torch.from_numpy(_rows(boxes, scores, labels)).to(cuda)
        fused, n = ops.wbf_3d(rows, torch.from_numpy(cnt).to(cuda), boxes.shape[0], tta.WBF_IOU_THR, tta.WBF_SKIP_BOX_THR)
        _wbf_check(fused[0].cpu().numpy(), n[0].item(), ref)
        outs.append((rows, cnt, fused, n))
    assert not np.any(tta_ref.wbf_3d(*cases[1][:3])['labels'] == 3)
    # three frames at once: each frame's single-frame result, bit for bit
    r1, r2 = outs[1], outs[2]
    K = r1[0].shape[1]
    rows = torch.cat([r1[0], r2[0], r1[0]])
    cnt = torch.from_numpy(np.concatenate([r1[1], r2[1], r1[1]])).to(cuda)
    fused, n = ops.wbf_3d(rows, cnt, 15, tta.WBF_IOU_THR, tta.WBF_SKIP_BOX_THR)
    for b, (_, _, f1, n1) in enumerate([r1, r2, r1]):
        assert torch.equal(n[b], n1[0]) and torch.equal(fused[b], f1[0])


def test_wbf_edge_cases(cuda):
    from detzero_b200 import ops
    from detzero_b200.det import tta
    boxes, scores, labels, counts = _random_views(3)
    rows = torch.from_numpy(_rows(boxes, scores, labels)).to(cuda)
    fused, n = ops.wbf_3d(rows, torch.zeros(15, dtype=torch.int32, device=cuda), 15, tta.WBF_IOU_THR, tta.WBF_SKIP_BOX_THR)
    assert n.item() == 0 and torch.all(fused == 0)
    # one view only: every surviving box is its own cluster (score / 1)
    one = rows[1:2]                                                    # a view without duplicate rows
    fused, n = ops.wbf_3d(one, torch.from_numpy(counts[1:2]).to(cuda), 1, tta.WBF_IOU_THR, tta.WBF_SKIP_BOX_THR)
    ref = tta_ref.wbf_3d(boxes[1:2], scores[1:2], labels[1:2])
    assert all(len(m) == 1 for m in ref['members'])
    _wbf_check(fused[0].cpu().numpy(), n[0].item(), ref)
    # the drop-in wbf_online
    b, s, l = tta.wbf_online(rows[..., :7], rows[..., 7:8], rows[..., 8:9])
    ref = tta_ref.wbf_3d(boxes, scores, labels)
    assert b.shape[0] == len(ref['scores']) and np.array_equal(l.cpu().numpy(), ref['labels'])


def _tta_model(cuda, tta):
    import bench
    from detzero_b200 import synthetic
    from detzero_b200.det import build_network
    from detzero_b200.det.dataset import SyntheticWaymoDataset, default_waymo_1sweep_cfg
    dcfg = default_waymo_1sweep_cfg()
    dcfg.POINT_CLOUD_RANGE = util.SMALL_RANGE
    dcfg.TTA = tta
    ds = SyntheticWaymoDataset(dcfg, util.CLASS_NAMES, training=False, num_frames=1, n_points=20000)
    cfg = synthetic.model_cfg('VoxelBackBone8x', 'tf32')
    cfg.BACKBONE_3D.COMPUTE_MODE = synthetic.DEFAULT_SP_MODE
    model = build_network(cfg, 3, ds).eval()
    weights.load_seeded(model, 21)
    bench.tune_head_for_bench(model)
    return ds, model.to(cuda)


def test_centerpoint_tta_end_to_end_and_graph(cuda):
    from detzero_b200.det import load_data_to_gpu
    ds, model = _tta_model(cuda, True)
    plain_ds, _ = _tta_model(cuda, False)
    clouds = [util.clustered_cloud(20000, 61, c=6), util.clustered_cloud(15000, 62, c=6)]
    items = [ds.process(ds.point_feature_encoder.forward({'points': p.copy(), 'frame_id': str(k)})) for k, p in enumerate(clouds)]
    batch = load_data_to_gpu(ds.collate_batch(items), cuda)
    V = len(NAMES)
    assert batch['tta_ops'] == NAMES and batch['batch_size'] == 2 * V
    with torch.no_grad():
        pred, _ = model(dict(batch))
        out = model.forward_device(dict(batch))
    assert len(pred) == 2
    vb, vc = out['tta_view_boxes_padded'].cpu().numpy(), out['tta_view_boxes_count'].cpu().numpy()
    fb, fc = out['final_boxes_padded'].cpu().numpy(), out['final_boxes_count'].cpu().numpy()
    multi = False
    for b, item in enumerate(items):
        # (a) per-view detections == the detector without TTA on the host-augmented, masked clouds
        views = tta_ref.augment(item['points'], NAMES)
        plain_items = [plain_ds.data_processor.forward({'points': q, 'frame_id': str(v)}) for v, q in enumerate(views)]
        with torch.no_grad():
            ref = model.forward_device(load_data_to_gpu(plain_ds.collate_batch(plain_items), cuda))
        rb, rc = ref['final_boxes_padded'].cpu().numpy(), ref['final_boxes_count'].cpu().numpy()
        assert np.array_equal(vc[b * V:(b + 1) * V], rc)
        for v in range(V):
            assert np.array_equal(vb[b * V + v, :rc[v]].view(np.uint32), rb[v, :rc[v]].view(np.uint32)), (b, v)
        assert rc.sum() > 0
        # (b) fused == oracle un-augment + WBF of those detections
        K = rb.shape[1]
        labels = np.where(np.arange(K)[None] < rc[:, None], rb[..., 8], 0).astype(np.int64)
        r = tta_ref.wbf_3d(tta_ref.unaugment(rb[..., :7], NAMES), rb[..., 7], labels)
        assert r['min_margin'] > 1e-5
        multi |= any(len(m) > 1 for m in r['members'])
        _wbf_check(fb[b], fc[b], r)
        assert pred[b]['pred_boxes'].shape[0] == fc[b]
    assert multi
    # CUDA-graph replay == eager, bit for bit
    g, static = model.capture_graph(dict(batch))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(static['final_boxes_count'], out['final_boxes_count'])
    assert torch.equal(static['final_boxes_padded'], out['final_boxes_padded'])
    assert torch.equal(static['tta_view_boxes_padded'], out['tta_view_boxes_padded'])


def test_tta_rejects_gather_slab(cuda):
    from detzero_b200.det import load_data_to_gpu
    ds, model = _tta_model(cuda, True)
    item = ds.process(ds.point_feature_encoder.forward({'points': util.clustered_cloud(5000, 1, c=6), 'frame_id': '0'}))
    batch = load_data_to_gpu(ds.collate_batch([item]), cuda)
    batch['gather_slab'] = None
    with pytest.raises(NotImplementedError):
        model.forward_device(batch)

"""Host restatement of CenterPoint test-time augmentation (oracle/tta_ref.py) against the reference's own outputs
(tests/golden/tta.npz, written by tests/golden/make_golden_tta.py), and the view list the product parses from the shipped config."""
import os

import numpy as np

from oracle import tta_ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'tta.npz')

REF_NAMES = ['tta_original', 'tta_flip_x', 'tta_flip_y', 'tta_flip_xy', 'tta_rot_-0.39365818', 'tta_rot_-0.78539816',
             'tta_rot_-1.17809724', 'tta_rot_-2.74889357', 'tta_rot_0.39365818', 'tta_rot_0.78539816', 'tta_rot_1.17809724',
             'tta_rot_2.74889357', 'tta_rot_3.14159265', 'tta_scale_0.95', 'tta_scale_1.05']


def _gold():
    return np.load(GOLD)


def test_augmented_points_bit_exact():
    g = _gold()
    names = [str(n) for n in g['names']]
    assert names == REF_NAMES
    aug = tta_ref.augment(g['points'], names)
    for v in range(len(names)):
        assert np.array_equal(aug[v].view(np.uint32), g['aug_points'][v].view(np.uint32)), names[v]


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) / np.maximum(np.abs(b), 1e-30)


def test_unaugment_and_fusion_match_reference():
    g = _gold()
    names = [str(n) for n in g['names']]
    un = tta_ref.unaugment(g['view_boxes'], names)
    valid = g['view_labels'] > 0
    assert np.all(_rel(un[valid], g['unaug_boxes'][valid])[np.abs(g['unaug_boxes'][valid]) > 1e-6] <= 1e-6)
    r = tta_ref.wbf_3d(un, g['view_scores'], g['view_labels'])
    assert r['boxes'].shape == g['fused_boxes'].shape
    assert np.array_equal(r['labels'], g['fused_labels'])
    assert np.all(np.abs(r['boxes'] - g['fused_boxes']) <= 1e-6 * np.maximum(np.abs(g['fused_boxes']), 1.0))
    assert np.all(_rel(r['scores'], g['fused_scores']) <= 1e-7)
    assert any(len(m) > 1 for m in r['members'])


def test_augmentor_parses_shipped_config():
    from detzero_b200.config import AttrDict, cfg_from_yaml_file
    from detzero_b200.det.dataset import default_waymo_1sweep_cfg
    from detzero_b200.det.tta import TestTimeAugmentor
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = cfg_from_yaml_file(os.path.join(here, 'detzero_b200', 'cfgs', 'det_dataset_cfgs', 'waymo_1sweep.yaml'), AttrDict())
    assert cfg.TTA is False and default_waymo_1sweep_cfg().TTA is False
    assert TestTimeAugmentor(cfg.TEST_TIME_AUGMENTOR).names == REF_NAMES
    assert TestTimeAugmentor(default_waymo_1sweep_cfg().TEST_TIME_AUGMENTOR).names == REF_NAMES


def test_tta_collate_keeps_original_points():
    from detzero_b200.det.dataset import SyntheticWaymoDataset, default_waymo_1sweep_cfg
    cfg = default_waymo_1sweep_cfg()
    cfg.TTA = True
    ds = SyntheticWaymoDataset(cfg, ['Vehicle', 'Pedestrian', 'Cyclist'], num_frames=2, n_points=5000)
    batch = ds.collate_batch([ds[0], ds[1]])
    assert batch['tta_ops'] == REF_NAMES and batch['batch_size'] == 2 * 15
    assert batch['points_per_frame'] == [5000, 5000] and batch['points'].shape[0] == 10000    # unmasked
    plain = SyntheticWaymoDataset(default_waymo_1sweep_cfg(), ['Vehicle', 'Pedestrian', 'Cyclist'], num_frames=1, n_points=5000)
    b0 = plain.collate_batch([plain[0]])
    assert 'tta_ops' not in b0 and b0['batch_size'] == 1

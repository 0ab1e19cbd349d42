"""Test-time augmentation of CenterPoint on the device.

``TestTimeAugmentor`` keeps the reference's name, constructor and view naming / order
(detection/detzero_det/datasets/augmentor/test_time_augmentor.py:9-100): ``tta_original``, then the flips, the rotations
(angle 0 skipped) and the scalings (1.0 skipped), in config order.  Instead of building the augmented copies in numpy in the
DataLoader workers it hands the per-view parameters to the device kernels (csrc/tta.cu): view expansion, box un-augmentation
(CenterPoint.test_time_augment, detection/detzero_det/models/centerpoint.py:131-208) and 3-D weighted box fusion
(``wbf_online``, detection/detzero_det/utils/ensemble_utils/ensemble.py:7-32)."""
import numpy as np
import torch

from .. import _lib, ops

#: ensemble.py:15-16, indexed by label - 1
WBF_IOU_THR = [0.8, 0.6, 0.7]
WBF_SKIP_BOX_THR = [0.1, 0.01, 0.01]


def _cos_sin_f32(angle):
    """cos / sin of float32(angle) in float32 torch on the CPU (common_utils.rotate_points_along_z: torch.from_numpy(...).float())"""
    a = torch.tensor([float(angle)], dtype=torch.float64).float()
    return float(torch.cos(a)[0]), float(torch.sin(a)[0]), float(a[0])


class TestTimeAugmentor:
    __test__ = False                                   # not a pytest class

    def __init__(self, augmentor_configs, logger=None):
        self.logger = logger
        cfg_list = augmentor_configs if isinstance(augmentor_configs, list) else augmentor_configs['AUG_CONFIG_LIST']
        disabled = [] if isinstance(augmentor_configs, list) else list(augmentor_configs.get('DISABLE_AUG_LIST', []))
        self.ops = [('tta_original', _lib_op('ORIGINAL'), 0.0)]
        for cur in cfg_list:
            if cur['NAME'] in disabled:
                continue
            self.ops.extend(getattr(self, cur['NAME'])(cur))

    # (name, op, parameter) per view, the reference's key names (test_time_augmentor.py:32-83)
    @staticmethod
    def world_flip(config):
        op = {'x': 'FLIP_X', 'y': 'FLIP_Y', 'xy': 'FLIP_XY'}
        return [('tta_flip_%s' % axis, _lib_op(op[axis]), 0.0) for axis in config['ALONG_AXIS_LIST']]

    @staticmethod
    def world_rotation(config):
        return [('tta_rot_%s' % str(a), _lib_op('ROT'), a) for a in config['ROT_ANGLE'] if a != 0.]

    @staticmethod
    def world_scaling(config):
        return [('tta_scale_%s' % str(s), _lib_op('SCALE'), s) for s in config['SCALE_RANGE'] if s != 1.]

    @property
    def names(self):
        return [n for n, _, _ in self.ops]

    def __len__(self):
        return len(self.ops)

    def expand_views(self):
        """(V, 4) float32 [op, p1, p2, p3] for dz_tta_expand: rotation by +a (cos, sin of float32(a)), scale by float32(s)"""
        rows = []
        for _, op, p in self.ops:
            if op == _lib.DZ_TTA_ROT:
                c, s, _ = _cos_sin_f32(p)
                rows.append([op, c, s, 0.0])
            else:
                rows.append([op, float(np.float32(p)), 0.0, 0.0])
        return np.asarray(rows, dtype=np.float32).reshape(-1, 4)

    def unaugment_views(self):
        """(V, 4) float32 for dz_tta_unaugment: rotation by -a plus heading offset float32(-a) (centerpoint.py:183-189)"""
        rows = []
        for _, op, p in self.ops:
            if op == _lib.DZ_TTA_ROT:
                c, s, a = _cos_sin_f32(-float(p))
                rows.append([op, c, s, a])
            else:
                rows.append([op, float(np.float32(p)), 0.0, 0.0])
        return np.asarray(rows, dtype=np.float32).reshape(-1, 4)

    def views_for(self, tta_ops):
        """check that a batch's ``tta_ops`` are this augmentor's views, in order"""
        if list(tta_ops) != self.names:
            raise ValueError('batch tta_ops %s do not match the TEST_TIME_AUGMENTOR views %s' % (list(tta_ops), self.names))
        return self


def _lib_op(name):
    return getattr(_lib, 'DZ_TTA_' + name)


def ops_from_names(tta_ops):
    """a TestTimeAugmentor equivalent to a batch's ``tta_ops`` list (the parameters are encoded in the names, as the reference
    parses them in centerpoint.py:165)"""
    aug = TestTimeAugmentor([])
    aug.ops = []
    for name in tta_ops:
        if name == 'tta_original':
            aug.ops.append((name, _lib.DZ_TTA_ORIGINAL, 0.0))
            continue
        _, kind, param = name.split('_', 2)
        if kind == 'flip':
            aug.ops.append((name, _lib_op({'x': 'FLIP_X', 'y': 'FLIP_Y', 'xy': 'FLIP_XY'}[param]), 0.0))
        elif kind == 'rot':
            aug.ops.append((name, _lib.DZ_TTA_ROT, float(param)))
        elif kind == 'scale':
            aug.ops.append((name, _lib.DZ_TTA_SCALE, float(param)))
        else:
            raise ValueError('unknown test-time augmentation %r' % name)
    return aug


def wbf_online(boxes, scores, labels, iou_thr=WBF_IOU_THR, skip_box_thr=WBF_SKIP_BOX_THR):
    """Device drop-in for ensemble_utils.ensemble.wbf_online: boxes (V, K, 7), scores (V, K, 1), labels (V, K, 1) of one frame,
    one "model" per view (rows with label 0 are padding) -> fused boxes (M, 7), scores (M,), labels (M,) in descending score
    order.  3-D IoU, conf_type 'avg', unit weights, allows_overflow False.  The counts are read back once to size the result."""
    V, K = boxes.shape[0], boxes.shape[1]
    dev = boxes.device
    rows = torch.cat([boxes[..., :7].float(), scores.reshape(V, K, 1).float(), labels.reshape(V, K, 1).float()], dim=2).contiguous()
    counts = torch.full((V,), K, dtype=torch.int32, device=dev)
    fused, n = ops.wbf_3d(rows, counts, V, iou_thr, skip_box_thr)
    m = int(n[0])
    out = fused[0, :m]
    return out[:, :7], out[:, 7], out[:, 8].long()

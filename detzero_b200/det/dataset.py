"""Data side of the hot path: the reference's DataProcessor / PointFeatureEncoder / collate contract
(detection/detzero_det/datasets/processor/data_processor.py:10-138, point_feature_encoder.py:4-57,
dataset.py:260-303) plus a synthetic Waymo-shape cloud source (there is no Waymo data or network here).

In this package voxelization is NOT done in DataLoader workers: ``transform_points_to_voxels`` only records the
grid (like the reference's ``..._placeholder`` step, data_processor.py:51-59) and the raw points go to the device,
where MeanVFE voxelizes them."""
from functools import partial

import numpy as np

from ..config import AttrDict
from .tta import TestTimeAugmentor


def mask_points_by_range(points, limit_range):
    """utils/detzero_utils/common_utils.py:247-250: x,y only, inclusive upper bound"""
    return (points[:, 0] >= limit_range[0]) & (points[:, 0] <= limit_range[3]) & \
           (points[:, 1] >= limit_range[1]) & (points[:, 1] <= limit_range[4])


class PointFeatureEncoder:
    """absolute_coordinates_encoding (point_feature_encoder.py:38-57): column select"""

    def __init__(self, config, point_cloud_range=None):
        self.cfg = config
        self.used = list(config.used_feature_list)
        self.src = list(config.src_feature_list)
        assert self.src[0:3] == ['x', 'y', 'z']
        self.point_cloud_range = point_cloud_range

    @property
    def num_point_features(self):
        return len(self.used)

    def forward(self, data_dict):
        pts = data_dict['points']
        cols = [pts[:, 0:3]] + [pts[:, self.src.index(x):self.src.index(x) + 1] for x in self.used if x not in 'xyz']
        data_dict['points'] = np.concatenate(cols, axis=1)
        data_dict['use_lead_xyz'] = True
        return data_dict


class DataProcessor:
    def __init__(self, processor_configs, point_cloud_range, training, num_point_features):
        self.point_cloud_range = np.asarray(point_cloud_range, dtype=np.float32)
        self.training = training
        self.num_point_features = num_point_features
        self.mode = 'train' if training else 'test'
        self.grid_size = self.voxel_size = None
        self.max_points_per_voxel, self.max_num_voxels = 5, 200000
        self.queue = [getattr(self, c.NAME)(config=c) for c in processor_configs]

    def mask_points_and_boxes_outside_range(self, data_dict=None, config=None):
        if data_dict is None:
            return partial(self.mask_points_and_boxes_outside_range, config=config)
        data_dict['points'] = data_dict['points'][mask_points_by_range(data_dict['points'], self.point_cloud_range)]
        return data_dict

    def shuffle_points(self, data_dict=None, config=None):
        if data_dict is None:
            return partial(self.shuffle_points, config=config)
        if config.SHUFFLE_ENABLED[self.mode]:
            data_dict['points'] = data_dict['points'][np.random.permutation(data_dict['points'].shape[0])]
        return data_dict

    def _grid(self, config):
        g = (self.point_cloud_range[3:6] - self.point_cloud_range[0:3]) / np.array(config.VOXEL_SIZE, dtype=np.float32)
        self.grid_size = np.round(g).astype(np.int64)
        self.voxel_size = list(config.VOXEL_SIZE)

    def transform_points_to_voxels_placeholder(self, data_dict=None, config=None):
        if data_dict is None:
            self._grid(config)
            return partial(self.transform_points_to_voxels_placeholder, config=config)
        return data_dict

    def transform_points_to_voxels(self, data_dict=None, config=None):
        """same YAML step name as the reference (data_processor.py:61-91); the voxel caps are recorded and the
        voxelization itself happens on the device in MeanVFE"""
        if data_dict is None:
            self._grid(config)
            self.max_points_per_voxel = int(config.MAX_POINTS_PER_VOXEL)
            self.max_num_voxels = int(config.MAX_NUMBER_OF_VOXELS[self.mode])
            return partial(self.transform_points_to_voxels, config=config)
        return data_dict

    def forward(self, data_dict, mask_range=True):
        """mask_range=False skips mask_points_and_boxes_outside_range: with test-time augmentation the reference masks each
        augmented view (dataset.py:240-246), and on the device the voxelizers drop exactly those points from each view"""
        for p in self.queue:
            if not mask_range and p.func.__name__ == 'mask_points_and_boxes_outside_range':
                continue
            data_dict = p(data_dict=data_dict)
        return data_dict


def synth_waymo_cloud(seed=0, n_target=180000, beams=64, azimuths=2650, sensor_h=2.0, sweep=0, ego_shift=0.0):
    """Waymo-shape 64-beam scan (SURVEY.md §8d config 2): ground plane at z=0, sensor 2 m up, random vertical
    obstacles at 8-75 m on 60 % of azimuths, sigma=2 cm range noise, second-return duplicates to reach n_target.
    Returns (n,6) f32 [x,y,z,intensity,elongation,offset] in the order a real frame file has
    (waymo_utils.py:284-302: NLZ column replaced by the 'offset' slot of src_feature_list)."""
    rng = np.random.default_rng(seed)
    az = np.linspace(-np.pi, np.pi, azimuths, endpoint=False)
    incl = np.linspace(np.deg2rad(-17.6), np.deg2rad(2.4), beams)
    A, I = np.meshgrid(az, incl, indexing='ij')
    with np.errstate(divide='ignore', invalid='ignore'):
        r_ground = np.where(I < 0, sensor_h / np.tan(-I), np.inf)
    has_obs = rng.random(azimuths) < 0.6
    obs_r = np.where(has_obs, rng.uniform(8, 75, azimuths), np.inf)
    obs_h = rng.uniform(0.5, 4.0, azimuths)
    R_obs = np.broadcast_to(obs_r[:, None], A.shape)
    z_at_obs = sensor_h + R_obs * np.tan(I)
    hit_obs = (z_at_obs >= 0) & (z_at_obs <= obs_h[:, None]) & np.isfinite(R_obs)
    r = np.where(hit_obs & (R_obs < r_ground), R_obs, r_ground)
    ok = np.isfinite(r) & (r < 75.0 * 1.4)
    r = np.where(ok, r, 0.0) + rng.normal(0, 0.02, r.shape)
    x = r * np.cos(A) + ego_shift
    y = r * np.sin(A)
    z = sensor_h + r * np.tan(I) - sensor_h          # vehicle frame: ground at z=0 -> shift so ground ~0
    z = np.where(hit_obs & (R_obs < r_ground), z_at_obs, 0.0) + rng.normal(0, 0.02, r.shape)
    pts = np.stack([x[ok], y[ok], z[ok]], axis=1)
    n = pts.shape[0]
    if n < n_target:                                   # second returns: jittered duplicates
        extra = pts[rng.integers(0, n, n_target - n)] + rng.normal(0, 0.03, (n_target - n, 3))
        pts = np.concatenate([pts, extra], axis=0)
        pts = pts[rng.permutation(pts.shape[0])]       # interleave like a real dual-return frame
    else:
        pts = pts[:n_target]
    inten = np.tanh(rng.uniform(0, 2, pts.shape[0]))
    elong = rng.uniform(0, 1, pts.shape[0])
    off = np.full(pts.shape[0], -0.1 * sweep)
    return np.concatenate([pts, inten[:, None], elong[:, None], off[:, None]], axis=1).astype(np.float32)


class SyntheticWaymoDataset:
    """DatasetTemplate-shaped source of synthetic frames: __getitem__ -> data_dict, collate_batch -> batch_dict with
    the reference's keys (dataset.py:260-303): points (N,1+C) [b,x,y,z,...], frame_id, batch_size (+ gt_boxes)."""

    def __init__(self, dataset_cfg, class_names, training=False, num_frames=8, n_points=180000, seed0=0):
        self.dataset_cfg = dataset_cfg
        self.class_names = class_names
        self.training = training
        self.tta = dataset_cfg.get('TTA', False)
        self.point_cloud_range = np.array(dataset_cfg.POINT_CLOUD_RANGE, dtype=np.float32)
        self.point_feature_encoder = PointFeatureEncoder(dataset_cfg.POINT_FEATURE_ENCODING, self.point_cloud_range)
        self.data_processor = DataProcessor(dataset_cfg.DATA_PROCESSOR, self.point_cloud_range, training,
                                            self.point_feature_encoder.num_point_features)
        self.grid_size = self.data_processor.grid_size
        self.voxel_size = self.data_processor.voxel_size
        self.max_points_per_voxel = self.data_processor.max_points_per_voxel
        self.max_num_voxels = self.data_processor.max_num_voxels
        self.num_frames, self.n_points, self.seed0 = num_frames, n_points, seed0
        tta_cfg = dataset_cfg.get('TEST_TIME_AUGMENTOR')
        self.test_time_augmentor = TestTimeAugmentor(tta_cfg) if tta_cfg is not None else None
        if self.tta and self.test_time_augmentor is None:
            raise ValueError('TTA: True needs a TEST_TIME_AUGMENTOR block in the dataset config')

    def __len__(self):
        return self.num_frames

    def __getitem__(self, index):
        pts = synth_waymo_cloud(self.seed0 + index, self.n_points)
        d = {'points': pts, 'frame_id': 'synth_%06d' % index, 'sequence_name': 'synthetic', 'sample_idx': index}
        d = self.point_feature_encoder.forward(d)
        return self.process(d)

    def process(self, data_dict):
        """the data processor; with TTA the original cloud stays unmasked and carries the view names (the views themselves are
        built on the device by CenterPoint)"""
        if not self.tta:
            return self.data_processor.forward(data_dict)
        data_dict = self.data_processor.forward(data_dict, mask_range=False)
        data_dict['tta_ops'] = self.test_time_augmentor.names
        return data_dict

    @staticmethod
    def collate_batch(batch_list):
        """dataset.py:260-303; with TTA (items carry ``tta_ops``) the points stay the B original frames, and the batch gets the
        view names and batch_size = B * views, as in the reference"""
        pts, sizes = [], []
        for b, d in enumerate(batch_list):
            p = d['points']
            pts.append(np.pad(p, ((0, 0), (1, 0)), mode='constant', constant_values=b))    # dataset.py:275-283
            sizes.append(p.shape[0])
        ret = {'points': np.concatenate(pts, axis=0).astype(np.float32), 'points_per_frame': sizes,
               'frame_id': np.array([d['frame_id'] for d in batch_list]), 'batch_size': len(batch_list)}
        if 'tta_ops' in batch_list[0]:
            ret['tta_ops'] = list(batch_list[0]['tta_ops'])
            ret['batch_size'] = len(batch_list) * len(ret['tta_ops'])
        return ret


def default_waymo_1sweep_cfg():
    """the dataset keys of detection/tools/cfgs/det_dataset_cfgs/waymo_1sweep.yaml that the hot path reads"""
    return AttrDict({
        'DATASET': 'SyntheticWaymoDataset',
        'POINT_CLOUD_RANGE': [-75.2, -75.2, -2, 75.2, 75.2, 4],
        'TTA': False,
        'TEST_TIME_AUGMENTOR': {
            'DISABLE_AUG_LIST': ['placeholder'],
            'AUG_CONFIG_LIST': [
                {'NAME': 'world_flip', 'ALONG_AXIS_LIST': ['x', 'y', 'xy']},
                {'NAME': 'world_rotation', 'ROT_ANGLE': [0, -0.39365818, -0.78539816, -1.17809724, -2.74889357, 0.39365818,
                                                         0.78539816, 1.17809724, 2.74889357, 3.14159265]},
                {'NAME': 'world_scaling', 'SCALE_RANGE': [0.95, 1.05]}]},
        'POINT_FEATURE_ENCODING': {'encoding_type': 'absolute_coordinates_encoding',
                                   'used_feature_list': ['x', 'y', 'z', 'intensity', 'elongation'],
                                   'src_feature_list': ['x', 'y', 'z', 'intensity', 'elongation', 'offset']},
        'DATA_PROCESSOR': [
            {'NAME': 'mask_points_and_boxes_outside_range', 'REMOVE_OUTSIDE_BOXES': True},
            {'NAME': 'shuffle_points', 'SHUFFLE_ENABLED': {'train': True, 'test': False}},
            {'NAME': 'transform_points_to_voxels', 'VOXEL_SIZE': [0.1, 0.1, 0.15], 'MAX_POINTS_PER_VOXEL': 5,
             'MAX_NUMBER_OF_VOXELS': {'train': 150000, 'test': 200000}}],
    })

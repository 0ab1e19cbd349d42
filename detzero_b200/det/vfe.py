"""Voxel feature encoders with the reference's names / ctor kwargs / batch_dict contract
(detection/detzero_det/models/centerpoint_modules/vfe.py:58-147), running on libdetzero_b200.

GPU ownership (SURVEY.md §8b): when the batch carries raw ``points`` (b,x,y,z,...) but no ``voxels`` (i.e. the data
processor used ``transform_points_to_voxels_placeholder``), ``MeanVFE`` runs the order-exact hard voxelizer on the
device, fused with the mean, and hands the level-0 grid index to the 3D backbone -- no CPU voxelization, no H2D of
8 MB of voxels, no host sync."""
import torch
import torch.nn as nn

from .. import ops
from ..spconv.utils import Point2VoxelGPU3d


class MeanVFE(nn.Module):
    def __init__(self, model_cfg, num_point_features, point_cloud_range=None, voxel_size=None, grid_size=None, **kwargs):
        super().__init__()
        self.model_cfg = model_cfg
        self.num_point_features = num_point_features
        self.point_cloud_range = None if point_cloud_range is None else [float(v) for v in point_cloud_range]
        self.voxel_size = None if voxel_size is None else [float(v) for v in voxel_size]
        # the voxel caps live in the DATA_PROCESSOR config in the reference (waymo_1sweep.yaml:76-82); CenterPoint
        # forwards them here because voxelization moved from the DataLoader workers to the device
        self.max_points = int(kwargs.get('max_points_per_voxel', 5))
        self.max_voxels = int(kwargs.get('max_num_voxels', 200000))
        self._gen = None

    def get_output_feature_dim(self):
        return self.num_point_features

    def _generator(self, device):
        if self._gen is None:
            self._gen = Point2VoxelGPU3d(self.voxel_size, self.point_cloud_range, self.num_point_features,
                                         self.max_points, self.max_voxels, device=device)
        return self._gen

    @torch.no_grad()
    def forward(self, batch_dict, **kwargs):
        if 'voxels' in batch_dict:
            # reference contract (vfe.py:66-83): voxels (M,P,C), voxel_num_points (M,)
            voxels = batch_dict['voxels'].float().contiguous()
            num = batch_dict['voxel_num_points'].int().contiguous()
            batch_dict['voxel_features'] = ops.mean_vfe(voxels, num)
            return batch_dict
        # device voxelization from the collated raw points (N, 1+C) [b,x,y,z,...] (dataset.py:275-283)
        points = batch_dict['points']
        B = int(batch_dict['batch_size'])
        gen = self._generator(points.device)
        if 'points_per_frame' in batch_dict:                     # host-side frame sizes: no sync needed
            sizes = [int(s) for s in batch_dict['points_per_frame']]
        else:
            sizes = torch.bincount(points[:, 0].long(), minlength=B).tolist()
        clouds, start = [], 0
        for s in sizes:
            clouds.append(points[start:start + s])
            start += s
        r = gen.voxelize_batch(clouds, xyz_off=1)
        batch_dict['voxels'] = r['voxels']
        batch_dict['voxel_num_points'] = r['num']
        batch_dict['voxel_coords'] = r['coords']
        batch_dict['voxel_features'] = r['mean']
        batch_dict['voxel_count'] = r['counters'][0:1]           # device scalar: true number of rows
        batch_dict['voxel_grid_index'] = r['index']
        batch_dict['voxel_wanted'] = (r['counters'][2:3], r['cap'], gen)      # checked in CenterPoint.post_processing
        return batch_dict


class DynamicMeanVFE(nn.Module):
    """vfe.py:86-147 -- dynamic voxelization: output ordered by key b*XYZ + x*YZ + y*Z + z (torch.unique order)."""

    def __init__(self, model_cfg, num_point_features, voxel_size, grid_size, point_cloud_range, **kwargs):
        super().__init__()
        self.model_cfg = model_cfg
        self.num_point_features = num_point_features
        self.grid_size = [int(g) for g in grid_size]              # x,y,z
        self.voxel_size = [float(v) for v in voxel_size]
        self.point_cloud_range = [float(v) for v in point_cloud_range]

    def get_output_feature_dim(self):
        return self.num_point_features

    #: capacity over the largest voxel count seen so far (the count is read back by CenterPoint.post_processing)
    CAP_HEADROOM = 1.3

    @torch.no_grad()
    def forward(self, batch_dict, **kwargs):
        points = batch_dict['points'].float().contiguous()       # (b, x, y, z, i, e, ...)
        B = int(batch_dict['batch_size'])
        c = points.shape[1] - 1
        # like the reference, a frame has no voxel limit: every voxel holds at least one point, so one row per point always holds
        # every voxel.  Once a count has been read back, the capacity follows it (smaller level-1 buffers and launch grids); a
        # frame with more voxels is reported as an overflow (never truncated silently), the hint grows and the frame is re-run.
        cap = points.shape[0]
        hint = getattr(self, '_cap_hint', None)
        if hint is not None:
            cap = min(cap, (int(hint * self.CAP_HEADROOM) + 127) // 128 * 128)
        cap = max(cap, 1)
        feats, coords, d_m = ops.voxelize_dynamic_mean(points, c, B, self.point_cloud_range, self.voxel_size,
                                                       self.grid_size, cap)
        batch_dict['voxel_features'] = feats
        batch_dict['voxel_coords'] = coords
        batch_dict['voxel_count'] = d_m
        batch_dict['voxel_wanted'] = (d_m, cap, self)            # checked in CenterPoint.post_processing
        return batch_dict

    def note_count(self, wanted, cap):
        """feed the read-back voxel count into the capacity hint; raises if the capacity truncated the frame"""
        self._cap_hint = max(int(wanted), int(getattr(self, '_cap_hint', 0) or 0))
        if wanted > cap:
            raise RuntimeError('voxel capacity overflow: %d voxels > capacity %d (hint raised; re-run the frame)' % (wanted, cap))

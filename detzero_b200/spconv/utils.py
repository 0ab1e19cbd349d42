"""GPU voxel generator with the constructor / call surface of ``spconv.utils.Point2VoxelCPU3d`` as used at
detection/detzero_det/datasets/processor/data_processor.py:70-83.

The reference creates the CPU generator lazily inside each DataLoader worker; this package instead keeps raw points
on the device (``transform_points_to_voxels_placeholder``, data_processor.py:51-59) and voxelizes in the main process
(SURVEY.md §8b "Ownership / threading").  Results are order-exact with the CPU generator (first-appearance voxel
ids, first ``max_num_points_per_voxel`` points per voxel in input order, voxel cap in appearance order)."""
import numpy as np
import torch

from .. import ops


class Point2VoxelGPU3d:
    def __init__(self, vsize_xyz, coors_range_xyz, num_point_features, max_num_points_per_voxel, max_num_voxels,
                 device='cuda'):
        self.vsize = [float(v) for v in vsize_xyz]
        self.range = [float(v) for v in coors_range_xyz]
        self.c = int(num_point_features)
        self.max_pts = int(max_num_points_per_voxel)
        self.max_voxels = int(max_num_voxels)
        g = np.round((np.asarray(self.range[3:6], np.float32) - np.asarray(self.range[0:3], np.float32)) /
                     np.asarray(self.vsize, np.float32)).astype(np.int64)
        self.grid_xyz = [int(v) for v in g]
        self.grid_zyx = self.grid_xyz[::-1]
        self.sparse_shape = [self.grid_zyx[0] + 1, self.grid_zyx[1], self.grid_zyx[2]]     # backbone3d.py:133
        self.device = torch.device(device)

    #: B > 1: one dz_voxelize_hard_batch call (frames overlapped on internal streams) instead of B sequential calls
    BATCHED = True

    def voxelize_batch(self, clouds, xyz_off=0):
        """clouds: list of (n_i, stride) float32 CUDA tensors (one per frame).  Returns capacity-sized tensors and
        device counters -- no host sync.  dict(voxels, coords[b,z,y,x], num, mean, counters, index, cap)"""
        B = len(clouds)
        cap = sum(min(int(c.shape[0]), self.max_voxels) for c in clouds)
        hint = getattr(self, '_cap_hint', None)           # largest voxel count seen so far (set by the caller's read-back)
        if hint is not None:
            cap = min(cap, (int(hint * 1.3) + 127) // 128 * 128)
        cap = max(cap, 1)
        dev = clouds[0].device
        voxels = torch.empty((cap, self.max_pts, self.c), dtype=torch.float32, device=dev)
        coords = torch.zeros((cap, 4), dtype=torch.int32, device=dev)
        num = torch.zeros((cap,), dtype=torch.int32, device=dev)
        mean = torch.empty((cap, self.c), dtype=torch.float32, device=dev)
        counters = torch.zeros(3, dtype=torch.int32, device=dev)
        index = ops.GridIndex(B, self.sparse_shape, dev, with_perm_cap=sum(int(c.shape[0]) for c in clouds) + 1)
        if B > 1 and self.BATCHED:
            ops.voxelize_hard_batch(clouds, xyz_off, self.c, self.range, self.vsize, self.grid_zyx, self.max_pts, self.max_voxels,
                                    voxels, coords, num, mean, counters, index)
        else:
            for b, pts in enumerate(clouds):
                ops.voxelize_hard(pts, xyz_off, self.c, self.range, self.vsize, self.grid_zyx, self.max_pts,
                                  self.max_voxels, b, voxels, coords, num, mean, counters, index)
        return dict(voxels=voxels, coords=coords, num=num, mean=mean, counters=counters, index=index, cap=cap)

    def note_count(self, wanted, cap):
        """feed the read-back voxel count into the capacity hint; raises if the capacity truncated the frame"""
        self._cap_hint = max(int(wanted), int(getattr(self, '_cap_hint', 0) or 0))
        if wanted > cap:
            raise RuntimeError('voxel capacity overflow: %d voxels > capacity %d (hint raised; re-run the frame)' % (wanted, cap))

    def point_to_voxel(self, points):
        """API-compatible single-cloud call: returns (voxels (M,P,C), coords (M,3) [z,y,x], num (M,)) CUDA tensors.
        Reads the voxel count back (one host sync) to slice the outputs like the CPU generator does."""
        if isinstance(points, np.ndarray):
            points = torch.from_numpy(np.ascontiguousarray(points, dtype=np.float32)).to(self.device)
        points = points.float().contiguous()
        r = self.voxelize_batch([points])
        m = int(r['counters'][0].item())
        self.note_count(int(r['counters'][2].item()), r['cap'])
        return r['voxels'][:m], r['coords'][:m, 1:4].contiguous(), r['num'][:m]


# the reference imports this name (data_processor.py:6); here it resolves to the GPU generator
Point2VoxelCPU3d = Point2VoxelGPU3d

"""``CenterPoint`` detector template + module registry (the reference's "Detector3DTemplate" role, SURVEY.md F2):
detection/detzero_det/models/centerpoint.py:15-129, models/__init__.py:8-29,
centerpoint_modules/__init__.py:8-17.  Modules are looked up by NAME from the YAML config exactly like the reference;
every module is ``forward(batch_dict) -> batch_dict``."""
import numpy as np
import torch
import torch.nn as nn

from . import backbone3d, dense, tta, vfe
from .. import ops

#: module registry, same keys as detzero_det.models.centerpoint_modules.__all__ (PDVHead = 2nd stage, out of scope)
cp_modules = {
    'MeanVFE': vfe.MeanVFE,
    'DynamicMeanVFE': vfe.DynamicMeanVFE,
    'VoxelBackBone8x': backbone3d.VoxelBackBone8x,
    'VoxelResBackBone8x': backbone3d.VoxelResBackBone8x,
    'HeightCompression': dense.HeightCompression,
    'BaseBEVBackbone': dense.BaseBEVBackbone,
    'CenterHead': dense.CenterHead,
}


class CenterPoint(nn.Module):
    def __init__(self, model_cfg, num_class, dataset):
        super().__init__()
        self.model_cfg = model_cfg
        self.num_class = num_class
        self.dataset = dataset
        self.tta = getattr(dataset, 'tta', False)
        self.class_names = dataset.class_names
        self.register_buffer('global_step', torch.LongTensor(1).zero_())
        self.second_stage = model_cfg.get('SECOND_STAGE', False)
        if self.second_stage:
            raise NotImplementedError('PDVHead second stage is out of scope (SURVEY.md §2.1)')
        self.module_list = self.build_networks()
        self._tta_views = {}                               # tta_ops names -> (expand, un-augment) view parameters

    @property
    def mode(self):
        return 'TRAIN' if self.training else 'TEST'

    def update_global_step(self):
        self.global_step += 1

    def build_networks(self):
        ds = self.dataset
        info = {'num_point_features': ds.point_feature_encoder.num_point_features, 'grid_size': ds.grid_size,
                'point_cloud_range': ds.point_cloud_range, 'voxel_size': ds.voxel_size}
        cfg = self.model_cfg
        m_vfe = cp_modules[cfg.VFE.NAME](model_cfg=cfg.VFE, num_point_features=info['num_point_features'],
                                         point_cloud_range=info['point_cloud_range'], voxel_size=info['voxel_size'],
                                         grid_size=info['grid_size'],
                                         max_points_per_voxel=getattr(ds, 'max_points_per_voxel', 5),
                                         max_num_voxels=getattr(ds, 'max_num_voxels', 200000))
        info['num_point_features'] = m_vfe.get_output_feature_dim()
        m_b3d = cp_modules[cfg.BACKBONE_3D.NAME](model_cfg=cfg.BACKBONE_3D, input_channels=info['num_point_features'],
                                                 grid_size=info['grid_size'], voxel_size=info['voxel_size'],
                                                 point_cloud_range=info['point_cloud_range'])
        info['num_point_features'] = m_b3d.num_point_features
        m_bev = cp_modules[cfg.MAP_TO_BEV.NAME](model_cfg=cfg.MAP_TO_BEV, grid_size=info['grid_size'])
        info['num_bev_features'] = m_bev.num_bev_features
        m_b2d = cp_modules[cfg.BACKBONE_2D.NAME](model_cfg=cfg.BACKBONE_2D, input_channels=info['num_bev_features'])
        info['num_bev_features'] = m_b2d.num_bev_features
        m_head = cp_modules[cfg.DENSE_HEAD.NAME](
            model_cfg=cfg.DENSE_HEAD, input_channels=info['num_bev_features'],
            num_class=self.num_class if not cfg.DENSE_HEAD.CLASS_AGNOSTIC else 1, class_names=self.class_names,
            grid_size=info['grid_size'], voxel_size=info['voxel_size'], point_cloud_range=info['point_cloud_range'],
            tta=self.tta, predict_boxes_when_training=self.second_stage)
        for name, m in (('vfe', m_vfe), ('backbone3d', m_b3d), ('map_to_bev', m_bev), ('backbone2d', m_b2d),
                        ('dense_head', m_head)):
            self.add_module(name, m)
        return [m_vfe, m_b3d, m_bev, m_b2d, m_head]

    def forward_device(self, batch_dict):
        """all device work of one batch, no host sync (capturable in a CUDA graph); result =
        batch_dict['final_boxes_padded'] (B,500,9) + ['final_boxes_count'] (B) + ['overflow_flag'] (1,) int32: number of
        sparse levels (and the voxelizer) whose true row count exceeded the capacity the kernels clamped to -- nonzero
        means rows were dropped and the step must be re-run with larger capacities (post_processing raises).

        With test-time augmentation (the batch carries the reference's ``tta_ops`` and ``batch_size`` = B*V) the B original frames
        are expanded into B*V views on the device, the modules run unchanged on them, and the final boxes are the per-frame
        weighted box fusion of the un-augmented views: (B, V*500, 9) + (B,).  The per-view result stays in
        ``tta_view_boxes_padded`` / ``tta_view_boxes_count``."""
        if 'tta_ops' in batch_dict:
            return self._forward_tta(batch_dict)
        for m in self.module_list:
            batch_dict = m(batch_dict)
        batch_dict['overflow_flag'] = self._overflow_flag(batch_dict)
        return batch_dict

    def _forward_tta(self, batch_dict):
        """CenterPoint.test_time_augment (detection/detzero_det/models/centerpoint.py:131-208) for B frames at once: each frame is
        fused on its own (the reference handles one frame per batch)"""
        if 'gather_slab' in batch_dict:
            raise NotImplementedError('test-time augmentation with the per-sequence box gather (gather_slab) is not supported')
        if len(self.dense_head.heads_list) != 1:
            raise NotImplementedError('test-time augmentation needs a single CenterHead head (got %d)' % len(self.dense_head.heads_list))
        names = tuple(batch_dict['tta_ops'])
        aug = self._tta_views.get(names)
        if aug is None:
            a = tta.ops_from_names(names)
            aug = self._tta_views[names] = (a.expand_views(), a.unaugment_views())
        V = len(names)
        BV = int(batch_dict['batch_size'])
        if BV % V:
            raise ValueError('batch_size %d is not a multiple of the %d test-time views' % (BV, V))
        B = BV // V
        points = batch_dict['points']
        if 'points_per_frame' in batch_dict:                     # host-side frame sizes: no sync needed
            sizes = [int(s) for s in batch_dict['points_per_frame']]
        else:
            sizes = torch.bincount(points[:, 0].long(), minlength=B).tolist()
        if len(sizes) != B:
            raise ValueError('points_per_frame has %d frames, tta batch_size %d / %d views = %d' % (len(sizes), BV, V, B))
        inner = {k: v for k, v in batch_dict.items() if k != 'tta_ops'}
        inner['points'] = ops.tta_expand(points.float().contiguous(), sizes, aug[0])
        inner['points_per_frame'] = [s for s in sizes for _ in range(V)]
        inner['batch_size'] = BV
        for m in self.module_list:
            inner = m(inner)
        view_boxes, view_counts = inner['final_boxes_padded'], inner['final_boxes_count']
        boxes = ops.tta_unaugment(view_boxes, view_counts, aug[1])
        fused, counts = ops.wbf_3d(boxes, view_counts, V, tta.WBF_IOU_THR, tta.WBF_SKIP_BOX_THR)
        out = dict(inner)
        out.update(points=points, points_per_frame=batch_dict.get('points_per_frame'), tta_ops=list(names), batch_size=B,
                   tta_view_boxes_padded=view_boxes, tta_view_boxes_count=view_counts,
                   final_boxes_padded=fused, final_boxes_count=counts)
        if out['points_per_frame'] is None:
            del out['points_per_frame']
        out['overflow_flag'] = self._overflow_flag(out)
        return out

    @staticmethod
    def _levels(batch_dict):
        levels = [t for t in batch_dict.get('multi_scale_3d_features', {}).values()] + [batch_dict.get('encoded_spconv_tensor')]
        return [t for t in levels if t is not None]

    def _overflow_flag(self, batch_dict):
        """device-side OR over every capacity-bounded count of the step (every kernel clamps with min(count, cap), so an
        overflow would otherwise truncate silently under CUDA-graph replay)"""
        flags = [(t._count > t._cap) for t in CenterPoint._levels(batch_dict)]
        vw = batch_dict.get('voxel_wanted')
        if vw is not None:
            flags.append(vw[0] > vw[1])
        if not flags:
            return torch.zeros(1, dtype=torch.int32, device=batch_dict['final_boxes_count'].device)
        return torch.cat([f.view(1) for f in flags]).sum(dtype=torch.int32).view(1)

    def capture_graph(self, batch_dict, warmup=2):
        """Capture forward_device for a fixed input shape in a CUDA graph (streams + graphs instead of a tracing compiler).
        ``batch_dict['points']`` becomes the static input buffer: copy new points into it, then ``replay()``.  Capacities
        must have settled (run a few frames through ``forward`` first: the capacity hints are read back there).
        Returns (graph, static_batch_dict_out)."""
        import torch
        static_in = dict(batch_dict)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s), torch.no_grad():
            for _ in range(warmup):
                self.forward_device(dict(static_in))
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(g):
            out = self.forward_device(dict(static_in))
        return g, out

    def forward(self, batch_dict):
        if self.training:
            raise NotImplementedError('training loop support is a next row (SURVEY.md §8f rank 1)')
        batch_dict = self.forward_device(batch_dict)
        return self.post_processing(batch_dict)

    def post_processing(self, batch_dict):
        """centerpoint.py:210-307 (single-stage branch): pred_dicts = final_box_dicts.  The recall bookkeeping
        (generate_recall_record) needs gt boxes + 3D IoU and only feeds a log line; it is reported as empty.
        This is the ONE device->host read of the step: box counts + the overflow flag + per-level site counts.  Works on
        the static output of a replayed CUDA graph as well: the counts are re-read on every call (never cached), every
        capacity hint is raised BEFORE an overflow is reported, and an overflow always raises (never truncates)."""
        counts = batch_dict['final_boxes_count']
        levels = CenterPoint._levels(batch_dict)
        vw = batch_dict.get('voxel_wanted')
        ovf = batch_dict.get('overflow_flag')
        parts = [counts.flatten().int()] + ([ovf] if ovf is not None else []) + [t._count for t in levels] + ([vw[0]] if vw is not None else [])
        flat = torch.cat(parts).tolist()
        nb = counts.numel()
        pos = nb
        flagged = 0
        if ovf is not None:
            flagged = int(flat[pos]); pos += 1
        over = []
        for t in levels:
            n = int(flat[pos]); pos += 1
            t._n = None
            try:
                t.set_num(n)                               # updates the producing layer's capacity hint, raises on overflow
            except RuntimeError as e:
                over.append(str(e))
                t._n = t._cap
        if vw is not None:
            try:
                vw[2].note_count(int(flat[pos]), vw[1])
            except RuntimeError as e:
                over.append(str(e))
        if over or flagged:
            raise RuntimeError('capacity overflow in %d place(s) (all hints raised; re-run the step, re-capture any CUDA graph): %s'
                               % (max(len(over), flagged), '; '.join(over) or 'device flag set'))
        shaped = torch.tensor(flat[:nb]).view(counts.shape)
        pred_dicts = dense.CenterHead.boxes_to_dicts(batch_dict['final_boxes_padded'], shaped)
        batch_dict['final_box_dicts'] = pred_dicts
        return pred_dicts, {}


def build_network(model_cfg, num_class, dataset):
    return {'CenterPoint': CenterPoint}[model_cfg.NAME](model_cfg=model_cfg, num_class=num_class, dataset=dataset)


def load_data_to_gpu(batch_dict, device='cuda'):
    """models/__init__.py:21-29 -- every ndarray -> float CUDA tensor (non_blocking from pinned memory)"""
    for key, val in batch_dict.items():
        if key in ('frame_id', 'metadata', 'sequence_name', 'pose', 'tta_ops', 'aug_matrix_inv', 'points_per_frame'):
            continue
        if isinstance(val, np.ndarray):
            batch_dict[key] = torch.from_numpy(val).float().to(device, non_blocking=True)
        elif isinstance(val, torch.Tensor) and not val.is_cuda:
            batch_dict[key] = val.float().to(device, non_blocking=True)
    return batch_dict

"""VoxelBackBone8x / VoxelResBackBone8x with the reference's module tree (=> identical state-dict keys), ctor kwargs
and batch_dict contract (detection/detzero_det/models/centerpoint_modules/backbone3d.py:64-338), on the sm_90a
sparse-conv kernels.  In eval mode every conv + BatchNorm1d + (bias) + (residual) + ReLU group is ONE launch."""
from functools import partial

import torch
import torch.nn as nn

from ..spconv import pytorch as spconv
from ..spconv.pytorch import fold_bn


def post_act_block(in_channels, out_channels, kernel_size, indice_key=None, stride=1, padding=0, conv_type='subm',
                   norm_fn=None, mode='fp32'):
    """backbone3d.py:64-83"""
    if conv_type == 'subm':
        conv = spconv.SubMConv3d(in_channels, out_channels, kernel_size, bias=False, indice_key=indice_key, mode=mode)
    elif conv_type == 'spconv':
        conv = spconv.SparseConv3d(in_channels, out_channels, kernel_size, stride=stride, padding=padding, bias=False,
                                   indice_key=indice_key, mode=mode)
    elif conv_type == 'inverseconv':
        conv = spconv.SparseInverseConv3d(in_channels, out_channels, kernel_size, indice_key=indice_key, bias=False)
    else:
        raise NotImplementedError
    return spconv.SparseSequential(conv, norm_fn(out_channels), nn.ReLU())


class SparseBasicBlock(spconv.SparseModule):
    """backbone3d.py:85-121: SubM(+bias) -> BN -> ReLU -> SubM(+bias) -> BN -> (+identity) -> ReLU"""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, norm_fn=None, downsample=None, indice_key=None, mode='fp32'):
        super().__init__()
        assert norm_fn is not None
        bias = norm_fn is not None
        self.conv1 = spconv.SubMConv3d(inplanes, planes, kernel_size=3, stride=stride, padding=1, bias=bias,
                                       indice_key=indice_key, mode=mode)
        self.bn1 = norm_fn(planes)
        self.relu = nn.ReLU()
        self.conv2 = spconv.SubMConv3d(planes, planes, kernel_size=3, stride=stride, padding=1, bias=bias,
                                       indice_key=indice_key, mode=mode)
        self.bn2 = norm_fn(planes)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        if self.training:                               # unfused, differentiable: conv -> BN (batch statistics) -> ReLU -> conv -> BN -> + x -> ReLU
            identity = x if self.downsample is None else self.downsample(x)
            out = self.conv1(x)
            out = out._like(self.relu(self.bn1(out._feat)))
            out = self.conv2(out)
            out = out._like(self.bn2(out._feat))
            return out._like(self.relu(out._feat + identity._feat))
        identity = x if self.downsample is None else self.downsample(x)
        s1, b1 = fold_bn(self.bn1, self.conv1.bias)
        out = self.conv1.forward_fused(x, s1, b1, None, True)
        s2, b2 = fold_bn(self.bn2, self.conv2.bias)
        return self.conv2.forward_fused(out, s2, b2, identity, True)


class _Backbone8xBase(nn.Module):
    def _input_tensor(self, batch_dict):
        feats, coords = batch_dict['voxel_features'], batch_dict['voxel_coords']
        if coords.dtype != torch.int32:
            coords = coords.int()
        return spconv.SparseConvTensor(features=feats, indices=coords, spatial_shape=self.sparse_shape,
                                       batch_size=batch_dict['batch_size'],
                                       count=batch_dict.get('voxel_count'), index=batch_dict.get('voxel_grid_index'))

    def _first_convs(self):
        """first conv of every indice_key, in execution order (the rulebook chain depends on coordinates only)"""
        seen, order = set(), []
        for m in self.modules():
            if isinstance(m, spconv._SparseConv) and m.indice_key not in seen:
                seen.add(m.indice_key)
                order.append(m)
        return order

    SIDE_STREAM_HIGH_PRIORITY = True

    def prebuild_rulebooks(self, x0):
        """Build all rulebooks of the frame on a side stream while the feature convolutions run on the main stream:
        rulebooks depend only on coordinates, so the whole chain (spconv2 -> subm2 -> spconv3 -> ...) can run ahead of the
        features.  Every conv waits on its own rulebook's event.  Captured as parallel branches by CUDA graphs."""
        main = torch.cuda.current_stream()
        if getattr(self, '_side', None) is None or self._side.device != x0._feat.device:
            # high priority: the short rulebook kernels must not queue behind the conv grids that fill every SM
            prio = -1 if self.SIDE_STREAM_HIGH_PRIORITY else 0
            self._side = torch.cuda.Stream(device=x0._feat.device, priority=prio)
            self._side2 = torch.cuda.Stream(device=x0._feat.device, priority=prio)
        side, side2 = self._side, self._side2
        side.wait_stream(main)
        side2.wait_stream(main)
        events = {}
        t = x0
        for conv in self._first_convs():
            with torch.cuda.stream(side):               # the coordinate chain: rulebook -> next level's sites -> rulebook ...
                rule = conv._rule(t, schedule=False)
                ev = torch.cuda.Event()
                ev.record(side)
            with torch.cuda.stream(side2):              # the tile schedules hang off the chain without lengthening it
                side2.wait_event(ev)
                conv._schedule(rule, t)
                ev2 = torch.cuda.Event()
                ev2.record(side2)
            events[conv.indice_key] = ev2
            if not conv.subm:                           # coordinates-only view of the strided conv's output sites
                with torch.cuda.stream(side):
                    t = spconv.SparseConvTensor(t._feat[:1].new_empty((rule.out_cap, 1)), rule.out_idx, rule.out_dhw, t.batch_size,
                                                indice_dict=t.indice_dict, count=rule.d_n_out, n_host=None, index=rule.out_index)
                t._producer = conv
        x0.indice_dict['__events__'] = events
        x0.indice_dict['__side__'] = (side, side2)

    def forward(self, batch_dict):
        x0 = self._input_tensor(batch_dict)
        if self.training:                               # training path: exact-size tensors, rulebooks inline (autograd, SURVEY.md §8f row 1)
            pass
        elif self.model_cfg.get('OVERLAP_RULEBOOKS', True) if hasattr(self.model_cfg, 'get') else True:
            self.prebuild_rulebooks(x0)
        x = self.conv_input(x0)
        x_conv1 = self.conv1(x)
        x_conv2 = self.conv2(x_conv1)
        x_conv3 = self.conv3(x_conv2)
        x_conv4 = self.conv4(x_conv3)
        out = self.conv_out(x_conv4)
        side = x0.indice_dict.pop('__side__', None)
        if side is not None:
            for s in side:
                torch.cuda.current_stream().wait_stream(s)           # join (all rulebook memory is safe to reuse afterwards)
            x0.indice_dict.pop('__events__', None)
        batch_dict.update({'encoded_spconv_tensor': out, 'encoded_spconv_tensor_stride': 8})
        batch_dict.update({'multi_scale_3d_features': {'x_conv1': x_conv1, 'x_conv2': x_conv2, 'x_conv3': x_conv3,
                                                       'x_conv4': x_conv4}})
        batch_dict.update({'multi_scale_3d_strides': {'x_conv1': 1, 'x_conv2': 2, 'x_conv3': 4, 'x_conv4': 8}})
        return batch_dict


class VoxelBackBone8x(_Backbone8xBase):
    """backbone3d.py:124-227"""

    def __init__(self, model_cfg, input_channels, grid_size, **kwargs):
        super().__init__()
        self.model_cfg = model_cfg
        ch = list(model_cfg.get('CHANNELS', [16, 32, 64, 128])) if hasattr(model_cfg, 'get') else [16, 32, 64, 128]
        mode = model_cfg.get('COMPUTE_MODE', 'fp32') if hasattr(model_cfg, 'get') else 'fp32'
        norm_fn = partial(nn.BatchNorm1d, eps=1e-3, momentum=0.01)
        gs = [int(g) for g in grid_size]
        self.sparse_shape = [gs[2] + 1, gs[1], gs[0]]
        block = partial(post_act_block, mode=mode)
        self.conv_input = spconv.SparseSequential(
            spconv.SubMConv3d(input_channels, ch[0], 3, padding=1, bias=False, indice_key='subm1', mode=mode),
            norm_fn(ch[0]), nn.ReLU())
        self.conv1 = spconv.SparseSequential(block(ch[0], ch[0], 3, norm_fn=norm_fn, padding=1, indice_key='subm1'))
        self.conv2 = spconv.SparseSequential(
            block(ch[0], ch[1], 3, norm_fn=norm_fn, stride=2, padding=1, indice_key='spconv2', conv_type='spconv'),
            block(ch[1], ch[1], 3, norm_fn=norm_fn, padding=1, indice_key='subm2'),
            block(ch[1], ch[1], 3, norm_fn=norm_fn, padding=1, indice_key='subm2'))
        self.conv3 = spconv.SparseSequential(
            block(ch[1], ch[2], 3, norm_fn=norm_fn, stride=2, padding=1, indice_key='spconv3', conv_type='spconv'),
            block(ch[2], ch[2], 3, norm_fn=norm_fn, padding=1, indice_key='subm3'),
            block(ch[2], ch[2], 3, norm_fn=norm_fn, padding=1, indice_key='subm3'),
            block(ch[2], ch[2], 3, norm_fn=norm_fn, padding=1, indice_key='subm3'))
        self.conv4 = spconv.SparseSequential(
            block(ch[2], ch[2], 3, norm_fn=norm_fn, stride=2, padding=(0, 1, 1), indice_key='spconv4', conv_type='spconv'),
            block(ch[2], ch[2], 3, norm_fn=norm_fn, padding=1, indice_key='subm4'),
            block(ch[2], ch[2], 3, norm_fn=norm_fn, padding=1, indice_key='subm4'),
            block(ch[2], ch[2], 3, norm_fn=norm_fn, padding=1, indice_key='subm4'))
        last_pad = model_cfg.get('last_pad', 0) if hasattr(model_cfg, 'get') else 0
        self.conv_out = spconv.SparseSequential(
            spconv.SparseConv3d(ch[2], ch[3], (3, 1, 1), stride=(2, 1, 1), padding=last_pad, bias=False,
                                indice_key='spconv_down2', mode=mode),
            norm_fn(ch[3]), nn.ReLU())
        self.num_point_features = ch[3]


class VoxelResBackBone8x(_Backbone8xBase):
    """backbone3d.py:231-338"""

    def __init__(self, model_cfg, input_channels, grid_size, **kwargs):
        super().__init__()
        self.model_cfg = model_cfg
        ch = list(model_cfg.get('CHANNELS', [16, 32, 64, 128])) if hasattr(model_cfg, 'get') else [16, 32, 64, 128]
        mode = model_cfg.get('COMPUTE_MODE', 'fp32') if hasattr(model_cfg, 'get') else 'fp32'
        norm_fn = partial(nn.BatchNorm1d, eps=1e-3, momentum=0.01)
        gs = [int(g) for g in grid_size]
        self.sparse_shape = [gs[2] + 1, gs[1], gs[0]]
        block = partial(post_act_block, mode=mode)
        Basic = partial(SparseBasicBlock, mode=mode)
        self.conv_input = spconv.SparseSequential(
            spconv.SubMConv3d(input_channels, ch[0], 3, padding=1, bias=False, indice_key='subm1', mode=mode),
            norm_fn(ch[0]), nn.ReLU())
        self.conv1 = spconv.SparseSequential(Basic(ch[0], ch[0], norm_fn=norm_fn, indice_key='res1'),
                                             Basic(ch[0], ch[0], norm_fn=norm_fn, indice_key='res1'))
        self.conv2 = spconv.SparseSequential(
            block(ch[0], ch[1], 3, norm_fn=norm_fn, stride=2, padding=1, indice_key='spconv2', conv_type='spconv'),
            Basic(ch[1], ch[1], norm_fn=norm_fn, indice_key='res2'), Basic(ch[1], ch[1], norm_fn=norm_fn, indice_key='res2'))
        self.conv3 = spconv.SparseSequential(
            block(ch[1], ch[2], 3, norm_fn=norm_fn, stride=2, padding=1, indice_key='spconv3', conv_type='spconv'),
            Basic(ch[2], ch[2], norm_fn=norm_fn, indice_key='res3'), Basic(ch[2], ch[2], norm_fn=norm_fn, indice_key='res3'))
        self.conv4 = spconv.SparseSequential(
            block(ch[2], ch[3], 3, norm_fn=norm_fn, stride=2, padding=(0, 1, 1), indice_key='spconv4', conv_type='spconv'),
            Basic(ch[3], ch[3], norm_fn=norm_fn, indice_key='res4'), Basic(ch[3], ch[3], norm_fn=norm_fn, indice_key='res4'))
        last_pad = model_cfg.get('last_pad', 0) if hasattr(model_cfg, 'get') else 0
        self.conv_out = spconv.SparseSequential(
            spconv.SparseConv3d(ch[3], ch[3], (3, 1, 1), stride=(2, 1, 1), padding=last_pad, bias=False,
                                indice_key='spconv_down2', mode=mode),
            norm_fn(ch[3]), nn.ReLU())
        self.num_point_features = ch[3]
        self.backbone_channels = {'x_conv1': ch[0], 'x_conv2': ch[1], 'x_conv3': ch[2], 'x_conv4': ch[3]}

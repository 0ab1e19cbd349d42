"""CPU restatement (torch-CPU / numpy) of the detector hot path, driven by a reference-shaped ``state_dict``
(TEST INFRASTRUCTURE -- see oracle/__init__.py).  Each function cites the reference lines it follows.  The restatement
is pinned by tests/golden (outputs of the reference's own modules run in the build container) -- tests/test_oracle.py.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import nms_bev_sorted
from . import spconv_ref as S


# ---------------------------------------------------------------------------------------------------------------
# VFE
# ---------------------------------------------------------------------------------------------------------------
def mean_vfe(voxels, num_points):
    """MeanVFE.forward, vfe.py:66-83"""
    v = torch.as_tensor(voxels, dtype=torch.float32)
    n = torch.as_tensor(num_points, dtype=torch.float32)
    return (v.sum(dim=1) / torch.clamp_min(n.view(-1, 1), 1.0)).contiguous()


def dynamic_mean_vfe(points, pc_range, voxel_size, grid_size):
    """DynamicMeanVFE.forward, vfe.py:110-147 (torch_scatter.scatter_mean == index_add sums / counts, SURVEY A.5).
    Keys are int64 here (the reference's int32 key overflows for batch index >= 24: a latent bug, SURVEY §8a a3)."""
    points = torch.as_tensor(points, dtype=torch.float32)
    rng = torch.tensor(pc_range, dtype=torch.float32)
    vs = torch.tensor(voxel_size, dtype=torch.float32)
    gs = torch.tensor(grid_size, dtype=torch.int32)
    pc = torch.floor((points[:, 1:4] - rng[0:3]) / vs).int()
    mask = ((pc >= 0) & (pc < gs)).all(dim=1)
    points, pc = points[mask], pc[mask].long()
    sxyz, syz, sz = int(gs[0] * gs[1] * gs[2]), int(gs[1] * gs[2]), int(gs[2])
    merge = points[:, 0].long() * sxyz + pc[:, 0] * syz + pc[:, 1] * sz + pc[:, 2]
    data = points[:, 1:].contiguous()
    unq, inv, cnt = torch.unique(merge, return_inverse=True, return_counts=True)
    sums = torch.zeros((unq.shape[0], data.shape[1]), dtype=torch.float32).index_add_(0, inv, data)
    mean = sums / cnt.view(-1, 1).float()
    coords = torch.stack((unq // sxyz, (unq % sxyz) // syz, (unq % syz) // sz, unq % sz), dim=1)
    coords = coords[:, [0, 3, 2, 1]].int()
    return mean.contiguous(), coords.contiguous()


# ---------------------------------------------------------------------------------------------------------------
# sparse backbone (backbone3d.py) -- functional over a state_dict
# ---------------------------------------------------------------------------------------------------------------
class SpT:
    def __init__(self, feats, idx, shape, B, cache=None):
        self.f, self.idx, self.shape, self.B = feats, np.asarray(idx), list(shape), B
        self.cache = cache if cache is not None else {}


def bn1d_eval(x, sd, p, eps=1e-3):
    """nn.BatchNorm1d(eps=1e-3) in eval mode (backbone3d.py:132,239)"""
    return (x - sd[p + '.running_mean']) / torch.sqrt(sd[p + '.running_var'] + eps) * sd[p + '.weight'] + sd[p + '.bias']


def sp_conv(t, sd, p, subm, ks, stride, pad, key):
    w = sd[p + '.weight']
    b = sd.get(p + '.bias')
    if subm:
        if key not in t.cache:
            t.cache[key] = S.rulebook_subm(t.idx, t.shape, ks)
        out = S.sparse_conv_native(t.f, w, t.cache[key], t.f.shape[0], b)
        return SpT(out, t.idx, t.shape, t.B, t.cache)
    if key not in t.cache:
        t.cache[key] = S.rulebook_conv(t.idx, t.shape, ks, stride, pad)
    oi, oshape, pairs = t.cache[key]
    out = S.sparse_conv_native(t.f, w, pairs, oi.shape[0], b)
    return SpT(out, oi, oshape, t.B, t.cache)


def post_act(t, sd, p, conv_type, ks, stride, pad, key):
    """post_act_block, backbone3d.py:64-83: conv -> BN -> ReLU"""
    o = sp_conv(t, sd, p + '.0', conv_type == 'subm', ks, stride, pad, key)
    o.f = torch.relu(bn1d_eval(o.f, sd, p + '.1'))
    return o


def basic_block(t, sd, p, key):
    """SparseBasicBlock.forward, backbone3d.py:105-121"""
    o = sp_conv(t, sd, p + '.conv1', True, 3, 1, 1, key)
    o.f = torch.relu(bn1d_eval(o.f, sd, p + '.bn1'))
    o = sp_conv(o, sd, p + '.conv2', True, 3, 1, 1, key)
    o.f = bn1d_eval(o.f, sd, p + '.bn2')
    o.f = torch.relu(o.f + t.f)
    return o


def voxel_backbone(sd, prefix, feats, coords, sparse_shape, B, res):
    """VoxelBackBone8x.forward (backbone3d.py:136-227) / VoxelResBackBone8x.forward (:243-338)"""
    P = prefix
    t = SpT(torch.as_tensor(feats, dtype=torch.float32), np.asarray(coords), sparse_shape, B)
    x = post_act(t, sd, P + 'conv_input', 'subm', 3, 1, 1, 'subm1')
    outs = {}
    if not res:
        x1 = post_act(x, sd, P + 'conv1.0', 'subm', 3, 1, 1, 'subm1')
        x2 = post_act(x1, sd, P + 'conv2.0', 'spconv', 3, 2, 1, 'spconv2')
        x2 = post_act(x2, sd, P + 'conv2.1', 'subm', 3, 1, 1, 'subm2')
        x2 = post_act(x2, sd, P + 'conv2.2', 'subm', 3, 1, 1, 'subm2')
        x3 = post_act(x2, sd, P + 'conv3.0', 'spconv', 3, 2, 1, 'spconv3')
        for i in (1, 2, 3):
            x3 = post_act(x3, sd, P + 'conv3.%d' % i, 'subm', 3, 1, 1, 'subm3')
        x4 = post_act(x3, sd, P + 'conv4.0', 'spconv', 3, 2, (0, 1, 1), 'spconv4')
        for i in (1, 2, 3):
            x4 = post_act(x4, sd, P + 'conv4.%d' % i, 'subm', 3, 1, 1, 'subm4')
    else:
        x1 = basic_block(basic_block(x, sd, P + 'conv1.0', 'res1'), sd, P + 'conv1.1', 'res1')
        x2 = post_act(x1, sd, P + 'conv2.0', 'spconv', 3, 2, 1, 'spconv2')
        x2 = basic_block(basic_block(x2, sd, P + 'conv2.1', 'res2'), sd, P + 'conv2.2', 'res2')
        x3 = post_act(x2, sd, P + 'conv3.0', 'spconv', 3, 2, 1, 'spconv3')
        x3 = basic_block(basic_block(x3, sd, P + 'conv3.1', 'res3'), sd, P + 'conv3.2', 'res3')
        x4 = post_act(x3, sd, P + 'conv4.0', 'spconv', 3, 2, (0, 1, 1), 'spconv4')
        x4 = basic_block(basic_block(x4, sd, P + 'conv4.1', 'res4'), sd, P + 'conv4.2', 'res4')
    out = post_act(x4, sd, P + 'conv_out', 'spconv', (3, 1, 1), (2, 1, 1), 0, 'spconv_down2')
    outs.update(x_conv1=x1, x_conv2=x2, x_conv3=x3, x_conv4=x4, out=out)
    return outs


def height_compression(t):
    """HeightCompression.forward, height_compression.py:20-25"""
    d = S.dense_from_sparse(t.f, t.idx, t.shape, t.B)
    N, C, D, H, W = d.shape
    return d.reshape(N, C * D, H, W)


# ---------------------------------------------------------------------------------------------------------------
# BEV backbone + CenterHead (backbone2d.py, center_head.py)
# ---------------------------------------------------------------------------------------------------------------
def bn2d_eval(x, sd, p, eps):
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'], sd[p + '.bias'],
                        False, 0.0, eps)


def bev_backbone(sd, prefix, x, layer_nums, layer_strides, upsample_strides):
    """BaseBEVBackbone.forward, backbone2d.py:89-120 (module indices from the constructor :32-81)"""
    ups = []
    for i in range(len(layer_nums)):
        p = '%sblocks.%d.' % (prefix, i)
        x = F.pad(x, (1, 1, 1, 1))                                                        # ZeroPad2d(1)
        x = torch.relu(bn2d_eval(F.conv2d(x, sd[p + '1.weight'], None, layer_strides[i], 0), sd, p + '2', 1e-3))
        for k in range(layer_nums[i]):
            c = 4 + 3 * k
            x = torch.relu(bn2d_eval(F.conv2d(x, sd[p + '%d.weight' % c], None, 1, 1), sd, p + '%d' % (c + 1), 1e-3))
        q = '%sdeblocks.%d.' % (prefix, i)
        s = upsample_strides[i]
        u = F.conv_transpose2d(x, sd[q + '0.weight'], None, stride=s)
        ups.append(torch.relu(bn2d_eval(u, sd, q + '1', 1e-3)))
    return torch.cat(ups, dim=1) if len(ups) > 1 else ups[0]


def center_head_maps(sd, prefix, x, head_names):
    """CenterHead.forward conv part, center_head.py:440-447 with SeparateHead (:14-48); BatchNorm2d default eps 1e-5"""
    p = prefix + 'shared_conv.'
    x = torch.relu(bn2d_eval(F.conv2d(x, sd[p + '0.weight'], sd.get(p + '0.bias'), 1, 1), sd, p + '1', 1e-5))
    out = {}
    for n in head_names:
        q = '%sheads_list.0.%s.' % (prefix, n)
        h = torch.relu(bn2d_eval(F.conv2d(x, sd[q + '0.0.weight'], sd.get(q + '0.0.bias'), 1, 1), sd, q + '0.1', 1e-5))
        out[n] = F.conv2d(h, sd[q + '1.weight'], sd[q + '1.bias'], 1, 1)
    return out


def _gather_feat(feat, ind):
    """centernet_utils.py:118-128"""
    dim = feat.size(2)
    ind = ind.unsqueeze(2).expand(ind.size(0), ind.size(1), dim)
    return feat.gather(1, ind)


def _transpose_and_gather_feat(feat, ind):
    """centernet_utils.py:131-135"""
    feat = feat.permute(0, 2, 3, 1).contiguous()
    feat = feat.view(feat.size(0), -1, feat.size(3))
    return _gather_feat(feat, ind)


def topk(scores, batch_iou, K):
    """_topk, centernet_utils.py:138-165"""
    batch, num_class, height, width = scores.size()
    scores = scores.flatten(2, 3)
    if batch_iou is not None:
        biou = torch.clamp(batch_iou.reshape(batch, 1, height * width), min=0, max=1)
        scores = scores * torch.pow(biou, 2)
    K1 = min(K, height * width)
    topk_scores, topk_inds = torch.topk(scores, K1)
    topk_inds = topk_inds % (height * width)
    topk_ys = torch.div(topk_inds, width, rounding_mode='trunc').float()
    topk_xs = (topk_inds % width).int().float()
    K2 = min(K, num_class * K1)
    topk_score, topk_ind = torch.topk(topk_scores.view(batch, -1), K2)
    topk_classes = torch.div(topk_ind, K1, rounding_mode='trunc').int()
    topk_inds = _gather_feat(topk_inds.view(batch, -1, 1), topk_ind).view(batch, K2)
    topk_ys = _gather_feat(topk_ys.view(batch, -1, 1), topk_ind).view(batch, K2)
    topk_xs = _gather_feat(topk_xs.view(batch, -1, 1), topk_ind).view(batch, K2)
    return topk_score, topk_inds, topk_classes, topk_ys, topk_xs


def decode_bbox_from_heatmap(maps, pc_range, voxel_size, fmap_stride, K, score_thresh, post_limit, use_iou):
    """CenterHead.generate_predicted_boxes (center_head.py:324-344) + decode_bbox_from_heatmap
    (centernet_utils.py:168-230)"""
    heatmap = maps['hm'].sigmoid()
    dim = maps['dim'].exp()
    rot_cos, rot_sin = maps['rot'][:, 0:1], maps['rot'][:, 1:2]
    batch_iou = maps['iou'] if use_iou else None
    B = heatmap.shape[0]
    scores, inds, class_ids, ys, xs = topk(heatmap, batch_iou, K)
    Kk = scores.shape[1]
    center = _transpose_and_gather_feat(maps['center'], inds).view(B, Kk, 2)
    rs = _transpose_and_gather_feat(rot_sin, inds).view(B, Kk, 1)
    rc = _transpose_and_gather_feat(rot_cos, inds).view(B, Kk, 1)
    cz = _transpose_and_gather_feat(maps['center_z'], inds).view(B, Kk, 1)
    dm = _transpose_and_gather_feat(dim, inds).view(B, Kk, 3)
    # float32 atan2 rounded once from float64: the correctly rounded heading, on every CPU.  torch's float32 atan2 kernels differ
    # by an ulp between its scalar and vectorised code paths, so a float32 call would tie the oracle to the CPU it runs on
    angle = torch.atan2(rs.double(), rc.double()).float()
    xs = xs.view(B, Kk, 1) + center[:, :, 0:1]
    ys = ys.view(B, Kk, 1) + center[:, :, 1:2]
    xs = xs * fmap_stride * voxel_size[0] + pc_range[0]
    ys = ys * fmap_stride * voxel_size[1] + pc_range[1]
    boxes = torch.cat((xs, ys, cz, dm, angle), dim=-1)
    lim = torch.tensor(post_limit, dtype=torch.float32)
    mask = (boxes[..., :3] >= lim[:3]).all(2) & (boxes[..., :3] <= lim[3:]).all(2)
    if score_thresh is not None:
        mask &= scores > score_thresh
    return [dict(pred_boxes=boxes[k, mask[k]], pred_scores=scores[k, mask[k]], pred_labels=class_ids[k, mask[k]])
            for k in range(B)]


def class_agnostic_nms(box_scores, box_preds, nms_thresh, pre_max, post_max):
    """model_nms_utils.class_agnostic_nms (:6-25) -> iou3d_nms_utils.nms_gpu (:154-170)"""
    if box_scores.shape[0] == 0:
        return torch.zeros(0, dtype=torch.long)
    s, indices = torch.topk(box_scores, k=min(pre_max, box_scores.shape[0]))
    boxes = box_preds[indices]
    order = s.sort(0, descending=True)[1]
    keep = torch.from_numpy(nms_bev_sorted(boxes[order][:, :7].numpy(), nms_thresh))
    return indices[order[keep][:post_max]]


def generate_predicted_boxes(maps, pc_range, voxel_size, fmap_stride, post_cfg, use_iou):
    """center_head.py:315-368 for one head with the identity class mapping; labels 1-based"""
    dicts = decode_bbox_from_heatmap(maps, pc_range, voxel_size, fmap_stride, post_cfg['MAX_OBJ_PER_SAMPLE'],
                                     post_cfg['SCORE_THRESH'], post_cfg['POST_CENTER_LIMIT_RANGE'], use_iou)
    out = []
    for d in dicts:
        sel = class_agnostic_nms(d['pred_scores'], d['pred_boxes'], post_cfg['NMS_THRESH'], post_cfg['NMS_PRE_MAXSIZE'],
                                 post_cfg['NMS_POST_MAXSIZE'])
        out.append(dict(pred_boxes=d['pred_boxes'][sel], pred_scores=d['pred_scores'][sel],
                        pred_labels=d['pred_labels'][sel].long() + 1))
    return out


def merge_sweeps(info, target_infos, points):
    """DatasetTemplate.merge_sweeps (detection/detzero_det/datasets/dataset.py:167-196), statement by statement: NLZ filter, tanh of
    the intensity, ego-motion transform through the float64 poses, time-offset column"""
    current_pose, current_time = info['pose'], info['time_stamp']
    clouds = []
    for i in range(len(target_infos)):
        cur = points[i]
        cur, nlz = cur[:, 0:5], cur[:, 5]
        cur = cur[nlz == -1]
        cur[:, 3] = np.tanh(cur[:, 3])
        T = np.linalg.inv(current_pose) @ target_infos[i]['pose']
        dt = int(target_infos[i]['time_stamp']) - int(current_time)
        cur[:, :3] = np.concatenate([cur[:, :3], np.ones((cur.shape[0], 1))], axis=1) @ T[:3, :].T
        clouds.append(np.concatenate([cur, float(dt) / 1000000. * np.ones((cur.shape[0], 1))], axis=1))
    return np.concatenate(clouds, axis=0)

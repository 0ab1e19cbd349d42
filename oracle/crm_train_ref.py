"""Float64 pure-PyTorch restatement of ConfidencePointnet's train-mode forward and loss (confidence_pointnet.py:80-150,
target_assign.py:55-70) on a state dict, with autograd doing the backward -- TEST INFRASTRUCTURE.

Token-major: every 1x1 conv is a matmul on (rows, C), every BatchNorm takes batch statistics over all rows (F.batch_norm, training),
which is what BatchNorm2d over (B, C, L, P) and BatchNorm1d over (B, C, L) compute."""
import numpy as np
import torch
import torch.nn.functional as F

EPS, MOMENTUM = 1e-3, 0.01
SCORE_THRESH = (0.35, 0.7)


def crm_train_iou(seed, B, L, box_num=None):
    """seeded per-box IoU labels on both sides of both thresholds, -1 past each track's box_num (WaymoConfidenceDataset's padding)"""
    g = np.random.default_rng([int(seed), 0xC12])
    # no value within 1e-3 of a threshold: 0.35 and 0.7 compare differently in float32 and float64
    iou = g.choice([0.0, 0.1, 0.3, 0.34, 0.36, 0.5, 0.69, 0.71, 0.85, 1.0, 1.2], size=(B, L))
    iou = iou + np.clip(g.normal(0, 0.02, (B, L)), -0.009, 0.009) * (g.random((B, L)) < 0.5)
    if box_num is None:
        box_num = g.integers(L // 2, L + 1, B)
    iou[np.arange(L)[None, :] >= np.asarray(box_num)[:, None]] = -1.0
    return torch.from_numpy(iou.astype(np.float32))


def _layer(x, sd, conv, bn, stats, relu=True):
    w = sd[conv + '.weight']
    x = x @ w.reshape(w.shape[0], -1).t()
    if conv + '.bias' in sd:
        x = x + sd[conv + '.bias']
    if bn is not None:
        x = F.batch_norm(x, stats[bn + '.running_mean'], stats[bn + '.running_var'], sd[bn + '.weight'], sd[bn + '.bias'],
                         training=True, momentum=MOMENTUM, eps=EPS)
        stats[bn + '.num_batches_tracked'] += 1
    return torch.relu(x) if relu else x


def crm_train_step(state_dict, conf_points, iou, score_thresh=SCORE_THRESH, device='cpu'):
    """one training forward + backward in float64.  state_dict: ConfidencePointnet keys (no 'reg.' prefix).  Returns (losses {name:
    float}, grads {param: tensor}, running stats after the step {buffer: tensor})"""
    sd = {k: v.to(device, torch.float64).clone().requires_grad_(True) for k, v in state_dict.items()
          if not k.endswith(('running_mean', 'running_var', 'num_batches_tracked'))}
    stats = {k: v.to(device).clone().double() if not k.endswith('num_batches_tracked') else v.to(device).clone()
             for k, v in state_dict.items() if k.endswith(('running_mean', 'running_var', 'num_batches_tracked'))}
    x = conf_points.to(device, torch.float64)
    B, L, P, C = x.shape
    x = x.reshape(B * L * P, C)
    e = 'pts_encoder_1.'
    y1 = _layer(x, sd, e + '0', e + '1', stats)
    y2 = _layer(y1, sd, e + '3', e + '4', stats)                     # the hook on pts_encoder_1[5]
    y3 = _layer(y2, sd, e + '6', e + '7', stats)
    E = y3.shape[1]
    g = y3.view(B * L, P, E).max(dim=1)[0]
    x4 = torch.cat([g.unsqueeze(1).expand(B * L, P, E), y2.view(B * L, P, -1)], dim=2).reshape(B * L * P, -1)
    y4 = _layer(x4, sd, 'pts_encoder_2.0', 'pts_encoder_2.1', stats)
    pool = y4.view(B * L, P, E).max(dim=1)[0]
    h = _layer(pool, sd, 'pts_mlp.0', 'pts_mlp.1', stats)
    tap = _layer(h, sd, 'pts_mlp.3', 'pts_mlp.4', stats)             # the hook on pts_mlp[5]
    gg = tap.view(B, L, E).max(dim=1)[0]
    h = torch.cat([gg.unsqueeze(1).expand(B, L, E), tap.view(B, L, E)], dim=2).reshape(B * L, 2 * E)
    h = _layer(h, sd, 'regression_mlp.0', 'regression_mlp.1', stats)
    out = _layer(h, sd, 'regression_mlp.3', 'regression_mlp.4', stats)
    preds = {}
    for t in ('score_reg', 'iou_reg'):
        hh = _layer(out, sd, 'heads.%s.0' % t, 'heads.%s.1' % t, stats)
        preds[t] = torch.sigmoid(_layer(hh, sd, 'heads.%s.3' % t, None, stats, relu=False)).reshape(-1)
    lab = torch.clamp(iou.to(device, torch.float64), 0, 1).reshape(-1)
    pos = lab >= score_thresh[1]
    mask = (lab < score_thresh[0]) | pos
    n = mask.sum()
    cls = F.binary_cross_entropy(preds['score_reg'][mask], pos.double()[mask], reduction='none').sum() / n
    iol = F.binary_cross_entropy(preds['iou_reg'][mask], lab[mask], reduction='none').sum() / n
    loss = cls + iol
    loss.backward()
    losses = {'bin_cls_loss': cls.item(), 'iou_loss': iol.item(), 'confidence_loss': loss.item()}
    return losses, {k: v.grad.detach() for k, v in sd.items()}, stats


def probe(name, shape, seed):
    """the seeded tensor a gradient that is not stored in full is dotted with"""
    from detzero_b200.synthetic import seeded_tensor
    return seeded_tensor('probe.' + name, shape, seed).double()

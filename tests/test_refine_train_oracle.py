"""The float64 restatement of CRM training (oracle/crm_train_ref.py) against the reference's own ConfidencePointnet
(tests/golden/crm_train.npz, made by tests/golden/make_golden_crm_train.py): losses, gradients and BatchNorm running statistics."""
import os

import numpy as np
import torch

from detzero_b200.refine.modules import ConfidencePointnet
from oracle import crm_train_ref, weights
from oracle import refine_inputs as ri

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'crm_train.npz')
SEED, B = 7301, 2


def test_restatement_matches_reference_golden():
    gold = np.load(GOLD)
    m = ConfidencePointnet(ri.crm_cfg(), 32, 32)
    sd = weights.load_seeded(m, SEED)
    pts = ri.crm_inputs(SEED, B=B)['conf_points']
    losses, grads, stats = crm_train_ref.crm_train_step(sd, pts, crm_train_ref.crm_train_iou(SEED, B, pts.shape[1]))
    for k, v in losses.items():
        assert abs(v - gold['loss.' + k]) <= 1e-12 * abs(gold['loss.' + k]), k
    # the gradient of pts_encoder_1.7.bias is 0 up to rounding (the crop sums of dz4 add up to 0 and g > 0 almost everywhere), so
    # the scale of a full gradient is floored at 1e-6 of the largest point-encoder gradient
    floor = 1e-6 * max(np.abs(gold[k]).max() for k in gold.files if k.startswith('grad.'))
    for k, g in grads.items():
        if 'grad.' + k in gold:
            ref = torch.from_numpy(gold['grad.' + k]).double()
            assert (g - ref).abs().max().item() <= 1e-6 * max(ref.abs().max().item(), floor), k     # the golden keeps fp32 copies
        else:
            assert abs((g * g).sum().item() - gold['gsq.' + k]) <= 1e-10 * gold['gsq.' + k], k
            p = crm_train_ref.probe(k, g.shape, SEED)
            assert abs((g * p).sum().item() - gold['gdot.' + k]) <= 1e-10 * (g.norm() * p.norm()).item(), k
    for k, v in stats.items():
        ref = torch.from_numpy(gold['bn.' + k])
        if k.endswith('num_batches_tracked'):
            assert int(v) == int(ref) == 1, k
        else:
            assert torch.allclose(v, ref.double(), rtol=1e-12, atol=1e-14), k


def test_pooling_at_the_argmax_rows_is_the_default_path():
    """pooled_rows at the float64 argmax of each crop and channel reproduces the max-pooled step bit for bit; record holds the
    inputs of both maxes and the pooled output"""
    m = ConfidencePointnet(ri.crm_cfg(), 32, 32)
    sd = weights.load_seeded(m, SEED)
    pts = ri.crm_inputs(SEED, B=B)['conf_points']
    iou = crm_train_ref.crm_train_iou(SEED, B, pts.shape[1])
    rec = {}
    losses, grads, stats = crm_train_ref.crm_train_step(sd, pts, iou, record=rec)
    crops, P = B * pts.shape[1], pts.shape[2]
    assert rec['enc1'].shape == rec['enc2'].shape == (crops, P, 256) and rec['pool'].shape == (crops, 256)
    assert torch.equal(rec['pool'], rec['enc2'].max(dim=1)[0])
    rows = {k: rec[k].max(dim=1)[1].int() for k in ('enc1', 'enc2')}
    l2, g2, s2 = crm_train_ref.crm_train_step(sd, pts, iou, pooled_rows=rows)
    assert l2 == losses
    for k in grads:
        assert torch.equal(g2[k], grads[k]), k
    for k in stats:
        assert torch.equal(s2[k], stats[k]), k
    # float32 autograd of the same forward runs and stays close to float64
    l32, g32, _ = crm_train_ref.crm_train_step(sd, pts, iou, pooled_rows=rows, dtype=torch.float32)
    assert all(g.dtype == torch.float32 for g in g32.values())
    for k, v in losses.items():
        assert abs(l32[k] - v) <= 1e-4 * abs(v), k

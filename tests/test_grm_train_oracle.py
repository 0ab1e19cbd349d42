"""The float64 restatement of GRM training (oracle/grm_train_ref.py) against the reference's own module (tests/golden/grm_train.npz,
made by tests/golden/make_golden_grm_train.py): losses, gradients and running statistics after one step, on the CPU."""
import os

import numpy as np
import torch

from detzero_b200.config import AttrDict
from detzero_b200.refine.modules import GeometryTransformer
from oracle import grm_train_ref, weights
from oracle import refine_inputs as ri

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'grm_train.npz')
SEED = 7411


def seeded_state_dict(seed=SEED):
    cfg = ri.grm_cfg()
    cfg.DECODER['dropout'] = 0.0
    m = GeometryTransformer(AttrDict(cfg), 11, 4)
    return weights.load_seeded(m, seed)


def test_restatement_matches_reference_golden():
    gold = np.load(GOLD)
    losses, grads, stats = grm_train_ref.grm_train_step(seeded_state_dict(), grm_train_ref.grm_train_inputs(SEED, 2))
    for k, v in losses.items():
        assert abs(v - gold['loss.' + k]) <= 1e-9 * abs(gold['loss.' + k]), k
    seen = set()
    for k, g in grads.items():
        if 'grad.' + k in gold:
            ref = torch.from_numpy(gold['grad.' + k]).double()          # stored as float32
            assert (g - ref).abs().max().item() <= 1e-6 * max(ref.abs().max().item(), 1e-6), k
        else:
            assert abs((g * g).sum().item() - gold['gsq.' + k]) <= 1e-9 * gold['gsq.' + k], k
            p = grm_train_ref.probe(k, g.shape, SEED)
            assert abs((g * p).sum().item() - gold['gdot.' + k]) <= 1e-9 * g.norm().item() * p.norm().item(), k
        seen.add(k)
    assert {k.split('.', 1)[1] for k in gold.files if k.startswith(('grad.', 'gsq.'))} == seen
    for k, v in stats.items():
        ref = torch.from_numpy(gold['bn.' + k])
        if k.endswith('num_batches_tracked'):
            assert int(v) == int(ref) == 1, k
        else:
            assert torch.allclose(v, ref.double(), rtol=1e-6, atol=1e-7), k


def test_pooling_at_the_argmax_rows_is_the_default_path():
    """pooled_rows at the float64 argmax of each group and channel reproduces the max-pooled step bit for bit (the device tests pool
    the restatement at the device's rows through this hook); record holds the inputs of both maxes"""
    B = 2
    sd = seeded_state_dict()
    inp = grm_train_ref.grm_train_inputs(SEED, B)
    rec = {}
    losses, grads, stats = grm_train_ref.grm_train_step(sd, inp, record=rec)
    Q, P = inp['geo_query_points'].shape[1:3]
    assert rec['memory'].shape == (B, 4096, 512) and rec['query'].shape == (B * Q, P, 256)
    rows = {k: rec[k].max(dim=1)[1].int() for k in ('memory', 'query')}
    l2, g2, s2 = grm_train_ref.grm_train_step(sd, inp, pooled_rows=rows)
    assert l2 == losses
    assert set(g2) == set(grads)
    for k in grads:
        assert torch.equal(g2[k], grads[k]), k
    for k in stats:
        assert torch.equal(s2[k], stats[k]), k


def test_targets_pick_the_nearest_anchor():
    gt = grm_train_ref.grm_train_gt(SEED, 4, 3)
    from detzero_b200.refine.modules import TargetAssigner
    ta = TargetAssigner(anchor_sizes=torch.tensor(grm_train_ref.ANCHORS), mode='geometry')
    t = ta.encode_torch({'gt_box': gt.reshape(-1, 7)})
    anchors = torch.tensor(grm_train_ref.ANCHORS)
    delta = (gt.reshape(-1, 7)[:, None, 3:6] - anchors) / anchors
    assert torch.equal(t['geometry_reg'], delta.reshape(-1, 9))
    assert torch.equal(t['geometry_cls'], delta.abs().sum(-1).argmin(-1))

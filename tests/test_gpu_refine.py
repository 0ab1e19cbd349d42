"""GPU parity tests for the refiner (GRM / PRM / CRM): product modules vs the golden outputs of the reference's own
modules (tests/golden/refine.npz, same seeded weights and inputs) and the attention kernel vs a plain PyTorch fp32
reference (floating-point kernel)."""
import os

import numpy as np
import pytest
import torch

from oracle import refine_inputs as ri
from oracle import weights
from tests import util
from detzero_b200 import _lib

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'refine.npz'))
SEED = 4321


def _to(d, dev):
    return {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


@pytest.mark.parametrize('Pq,Pk,masked', [(200, 200, True), (200, 9600, True), (3, 4096, False), (77, 130, True)])
def test_attention_vs_torch(cuda, Pq, Pk, masked):
    """attention logits / outputs: fp32 tolerance 1e-4 rel (SURVEY.md §8c)"""
    from detzero_b200 import ops
    g = torch.Generator().manual_seed(Pq + Pk)
    B, H, dh = 3, 8, 32
    q = torch.randn(B, Pq, H * dh, generator=g) * 0.5
    k = torch.randn(B, Pk, H * dh, generator=g)
    v = torch.randn(B, Pk, H * dh, generator=g)
    mask = torch.zeros(B, Pk, dtype=torch.bool)
    if masked:
        for b in range(B):
            mask[b, int(Pk * (0.3 + 0.3 * b)):] = True
    qh, kh, vh = [t.view(B, -1, H, dh).permute(0, 2, 1, 3) for t in (q, k, v)]
    s = qh @ kh.transpose(-1, -2)
    s = s.masked_fill(mask[:, None, None, :], float('-inf'))
    ref = (torch.softmax(s, dim=-1) @ vh).permute(0, 2, 1, 3).reshape(B, Pq, H * dh)
    for mode, tol in ((_lib.DZ_F32, 1e-4), (_lib.DZ_TF32, 3e-3)):
        out = ops.attention(q.to(cuda), k.to(cuda), v.to(cuda), mask.to(torch.uint8).to(cuda) if masked else None, H, mode=mode)
        assert util.rel_err(out.cpu(), ref) < tol, mode


def test_linear_layernorm_groupmax(cuda):
    from detzero_b200 import ops
    g = torch.Generator().manual_seed(0)
    for M, K, N in [(1000, 32, 128), (513, 11, 128), (200, 4, 256), (77, 384, 512)]:
        x, w = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * 0.2
        sc, sh = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g)
        ref = torch.relu((x @ w.t()) * sc + sh)
        out = ops.linear(x.to(cuda), w.to(cuda), sc.to(cuda), sh.to(cuda), True)
        assert util.rel_err(out.cpu(), ref) < 1e-5
        out = ops.linear(x.to(cuda), ops.round_tf32(w).to(cuda), sc.to(cuda), sh.to(cuda), True, mode=_lib.DZ_TF32)
        assert util.rel_err(out.cpu(), ref) < 2e-3
    x, r = torch.randn(300, 256, generator=g), torch.randn(300, 256, generator=g)
    ln = torch.nn.LayerNorm(256)
    ln.weight.data = torch.rand(256, generator=g) + 0.5
    ln.bias.data = torch.randn(256, generator=g)
    out = ops.layernorm_residual(x.to(cuda), r.to(cuda), ln.weight.data.to(cuda), ln.bias.data.to(cuda), ln.eps)
    assert util.rel_err(out.cpu(), ln(x + r).detach()) < 1e-5
    y = ops.group_max(x.to(cuda), 30, 10)
    assert torch.equal(y.cpu(), x.view(30, 10, 256).max(dim=1)[0])


@pytest.mark.parametrize('mode,tol', [('fp32', 1e-3), ('tf32', 3e-2)])
def test_prm_vs_reference_golden(cuda, mode, tol):
    from detzero_b200.refine import PositionTransformer
    cfg = ri.prm_cfg()
    cfg.COMPUTE_MODE = mode
    m = PositionTransformer(cfg, 32, 32).eval()
    weights.load_seeded(m, SEED)
    m = m.to(cuda)
    d = m(_to(ri.prm_inputs(SEED), cuda))
    assert util.rel_err(d['query'].cpu(), GOLD['prm.query']) < (1e-4 if mode == 'fp32' else 5e-3)
    s = GOLD['prm.memory_sum']
    assert abs(d['memory'].double().abs().sum().item() - s[1]) < (1e-4 if mode == 'fp32' else 2e-3) * s[1]
    valid = (ri.prm_inputs(SEED)['padding_mask'] == 0)
    for k in ('center_reg', 'heading_cls', 'heading_reg'):
        got, want = m.preds_dict[k].cpu(), torch.from_numpy(GOLD['prm.' + k])
        assert util.rel_err(got[valid], want[valid]) < tol, k          # padded boxes attend to nothing meaningful
    got, want = d['batch_box_preds'].cpu(), torch.from_numpy(GOLD['prm.batch_box_preds'])
    assert (got[valid][:, :6] - want[valid][:, :6]).abs().max().item() < tol     # refined boxes <= 1e-3 in fp32 (SURVEY §8c)


@pytest.mark.parametrize('mode,tol', [('fp32', 1e-3), ('tf32', 3e-2)])
def test_grm_vs_reference_golden(cuda, mode, tol):
    """fp32: the exact-FMA kernels; tf32: the wgmma linears + attention the production configuration runs"""
    from detzero_b200.refine import GeometryTransformer
    cfg = ri.grm_cfg()
    cfg.COMPUTE_MODE = mode
    m = GeometryTransformer(cfg, 11, 4).eval()
    weights.load_seeded(m, SEED + 1)
    m = m.to(cuda)
    d = m(_to(ri.grm_inputs(SEED + 1), cuda))
    assert util.rel_err(m.preds_dict['geometry_cls'].cpu(), GOLD['grm.geometry_cls']) < tol
    assert util.rel_err(m.preds_dict['geometry_reg'].cpu(), GOLD['grm.geometry_reg']) < tol
    assert (d['batch_box_preds'].cpu() - torch.from_numpy(GOLD['grm.batch_box_preds'])).abs().max().item() < (1e-3 if mode == 'fp32' else 0.1)    # reg * anchor (<= 10 m)


@pytest.mark.parametrize('mode,tol', [('fp32', 1e-4), ('tf32', 5e-3)])
def test_crm_vs_reference_golden(cuda, mode, tol):
    from detzero_b200.refine import ConfidencePointnet
    cfg = ri.crm_cfg()
    cfg.COMPUTE_MODE = mode
    m = ConfidencePointnet(cfg, 32, 32).eval()
    weights.load_seeded(m, SEED + 2)
    m = m.to(cuda)
    d = m(_to(ri.crm_inputs(SEED + 2), cuda))
    assert (d['pred_score'].cpu() - torch.from_numpy(GOLD['crm.pred_score'])).abs().max().item() < tol


def test_grouped_linear_and_fused_maxpool(cuda):
    """dz_linear_fwd_grouped == Linear(cat([global.expand, per-row])) and dz_linear_max_fwd == max over groups of Linear(...):
    the two PointNet fusions of the refiner, against plain PyTorch fp32"""
    from detzero_b200 import ops
    g = torch.Generator().manual_seed(7)
    G, gsize, Cg, Cp, N = 5, 384, 256, 128, 512
    glob, per = torch.randn(G, Cg, generator=g), torch.randn(G * gsize, Cp, generator=g)
    w = torch.randn(N, Cg + Cp, generator=g) * 0.05
    sc, sh = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1
    cat = torch.cat([glob[:, None, :].expand(G, gsize, Cg), per.view(G, gsize, Cp)], dim=2).reshape(G * gsize, -1)
    ref = torch.relu((cat @ w.t()) * sc + sh)
    for mode, tol in ((_lib.DZ_F32, 1e-5), (_lib.DZ_TF32, 3e-3)):
        rnd = ops.round_tf32 if mode == _lib.DZ_TF32 else (lambda t: t)
        gshift = ops.linear(glob.to(cuda), rnd(w[:, :Cg].contiguous()).to(cuda), sc.to(cuda), None, False, mode=mode)
        out = ops.linear_grouped(per.to(cuda), rnd(w[:, Cg:].contiguous()).to(cuda), gshift, gsize, sc.to(cuda), sh.to(cuda), True, mode=mode)
        assert util.rel_err(out.cpu(), ref) < tol, mode
    # fused last layer + max over the points of a crop (group = 256 rows), incl. a group count that leaves a partial last CTA wave
    for G2, group in ((37, 256), (3, 4096)):
        x = torch.randn(G2 * group, 128, generator=g)
        w2 = torch.randn(256, 128, generator=g) * 0.1
        sc2, sh2 = torch.rand(256, generator=g) + 0.5, torch.randn(256, generator=g)
        for relu in (True, False):
            y = (x @ w2.t()) * sc2 + sh2
            ref2 = (torch.relu(y) if relu else y).view(G2, group, 256).max(dim=1)[0]
            out = ops.linear_max(x.to(cuda), ops.round_tf32(w2).to(cuda), group, sc2.to(cuda), sh2.to(cuda), relu, mode=_lib.DZ_TF32)
            assert util.rel_err(out.cpu(), ref2) < 3e-3, (G2, group, relu)

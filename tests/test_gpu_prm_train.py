"""One PRM training step on the device (PositionTransformer.forward_train / get_loss: the query encoder and the memory path on the
train-mode point layers of csrc/pointmlp_train.cu, the rest through autograd) against the plain-PyTorch autograd restatement of
the reference's forward and loss (tests/prm_train_ref.py) run in float64 on a copy of the same module.

Bounds, the GRM step's (tests/test_gpu_grm_train.py).  fp32: 1e-5 relative on every loss; per parameter, the largest gradient
error within 1e-4 of the parameter's largest gradient (floored at FLOOR times the largest gradient of the model), or within
K = 32 times the error float32 autograd of the same tree makes on the same batch, whichever is larger (the second term covers
gradients that are a small remainder of large cancelling terms: the memory path sums B * L * 48 rows whose terms cancel through
the softmax and BatchNorm backwards; K is stated below).  tf32: 5e-3 relative on the losses and 1e-2 on the gradients (the
GRM step's derivation: 2^-10 per TF32 layer, ten layers forward and backward), or K times the error of float32 autograd with TF32
matmuls and convolutions on the same batch."""
import copy

import numpy as np
import pytest
import torch

from detzero_b200.config import AttrDict
from detzero_b200.refine.modules import RefineTemplate
from detzero_b200.synthetic import load_seeded, prm_cfg
from tests import prm_train_ref as PR

pytestmark = pytest.mark.gpu
L, P, PM, C = 200, 256, 48, 32
# K is measured, not derived: with the GRM step's ASSOC = 8 two fp32 gradients went over, at 9.2 times the float32 autograd error
# (memory_mlp.0.weight, B = 2: its per-track parts are sums over L * 48 = 9600 cancelling rows, where the GRM sums 4096) and 15.5
# times (query_encoder.4.bias, B = 8: a BatchNorm bias whose gradient is 0 up to rounding, 7e-6 absolute); 32 leaves room for
# another batch
K = 32
# BatchNorm biases whose output reaches the loss only through another conv + BatchNorm have a gradient that is 0 up to rounding (its
# rows add up to 0), so, as in tests/test_gpu_grm_train.py, every gradient's scale is floored at FLOOR times the largest gradient
FLOOR = 1e-2


def model(mode, dropout=0.0, seed=5):
    cfg = prm_cfg()
    cfg.COMPUTE_MODE = mode
    cfg.DECODER['dropout'] = dropout
    m = RefineTemplate(AttrDict({'NAME': 'PositionRefineModel', 'QUERY_POINT_DIMS': C, 'MEMORY_POINT_DIMS': C, 'REGRESSION': cfg}))
    load_seeded(m.reg, seed)
    return m.cuda().train()


def batch(B, seed=0):
    """B tracks of L slots, box_num spread over 1..L, padded boxes zero rows, points near the boxes, ground truth near the boxes with
    headings across +-pi (one exactly at float32 pi)"""
    g = torch.Generator(device='cuda').manual_seed(seed)
    box_num = torch.tensor([L] + [int(x) for x in np.random.default_rng(seed).integers(1, L, B - 1)], dtype=torch.int32)[:B]
    valid = (torch.arange(L)[None] < box_num[:, None]).cuda()
    traj = torch.zeros(B, L, 7, device='cuda')
    traj[..., 0] = torch.linspace(-20, 20, L, device='cuda')
    traj[..., 1:3] = 0.3 * torch.randn(B, L, 2, device='cuda', generator=g)
    traj[..., 3:6] = torch.tensor([4.5, 1.9, 1.6], device='cuda')
    traj[..., 6] = 0.2 * torch.randn(B, L, device='cuda', generator=g)
    gt = traj.clone()
    gt[..., :3] += 0.2 * torch.randn(B, L, 3, device='cuda', generator=g)
    gt[..., 6] = (torch.rand(B, L, device='cuda', generator=g) * 2 - 1) * np.pi
    gt[0, 0, 6] = float(np.float32(np.pi))
    q = torch.randn(B, L, P, C, device='cuda', generator=g)
    m = torch.randn(B, L, PM, C, device='cuda', generator=g)
    v4 = valid[:, :, None, None]
    return {'pos_query_points': q * v4, 'pos_memory_points': m * v4, 'pos_trajectory': traj * valid[..., None],
            'gt_pos_trajectory': gt * valid[..., None], 'padding_mask': (~valid).float(), 'box_num': box_num.cuda(),
            'pos_init_box': torch.zeros(B, 7, device='cuda')}


def device_step(m, d):
    m.zero_grad(set_to_none=True)
    ret, tb, _ = m(dict(d))
    ret['loss'].backward()
    return {k: float(v) for k, v in tb.items()}, {n: p.grad.detach().clone() for n, p in m.reg.named_parameters() if p.grad is not None}


def _autograd32(reg, d, tf32):
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    try:
        return PR.step(reg, d, torch.float32)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
@pytest.mark.parametrize('B', [2, 8])
def test_step_matches_float64_restatement(cuda, mode, B):
    m = model(mode)
    d = batch(B, seed=B)
    ref0 = copy.deepcopy(m.reg)                                      # the state before the step (BatchNorm running stats move)
    loss, grads = device_step(m, d)
    rl, rg = PR.step(ref0, d, torch.float64)
    _, g32 = _autograd32(ref0, d, mode == 'tf32')
    assert set(grads) == set(rg), set(grads) ^ set(rg)
    ltol, gtol = (1e-5, 1e-4) if mode == 'fp32' else (5e-3, 1e-2)
    for k in ('center_reg_loss', 'heading_cls_loss', 'heading_reg_loss', 'position_loss'):
        assert abs(loss[k] - rl[k]) <= ltol * abs(rl[k]), (k, loss[k], rl[k])
    assert loss['full_loss'] == loss['position_loss']
    worst = []
    largest = max(r.abs().max().item() for r in rg.values())
    for n, r in rg.items():
        err = (grads[n].double() - r).abs().max().item()
        scale = max(r.abs().max().item(), FLOOR * largest)
        bound = max(gtol * scale, K * (g32[n].double() - r).abs().max().item())
        worst.append((err / bound, n))
        assert err <= bound, (n, err, bound)
    print(mode, B, 'worst gradient error / bound: %.3g (%s)' % max(worst))


def test_determinism_dropout_and_refusal(cuda):
    d = batch(4, seed=3)
    a, ga = device_step(model('tf32'), d)
    b, gb = device_step(model('tf32'), d)
    assert a == b and all(torch.equal(ga[n], gb[n]) for n in ga)
    c, gc = device_step(model('tf32', dropout=0.1), d)
    assert c['position_loss'] != a['position_loss'] and np.isfinite(c['position_loss'])
    assert all(bool(torch.isfinite(v).all()) for v in gc.values())
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        with pytest.raises(RuntimeError, match='allow_tf32'):
            model('fp32')(dict(d))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def test_shape_and_width_rejections(cuda):
    d = batch(2)
    bad = dict(d, pos_memory_points=d['pos_memory_points'][:, :, :32])
    with pytest.raises(ValueError, match='48'):
        model('tf32')(bad)
    bad = dict(d, pos_query_points=d['pos_query_points'][:, :, :100])
    with pytest.raises(ValueError, match='multiple of 64'):
        model('tf32')(bad)
    cfg = prm_cfg()
    cfg.QUERY_ENCODER = [96, 128]
    cfg.COMPUTE_MODE = 'tf32'
    m = RefineTemplate(AttrDict({'NAME': 'PositionRefineModel', 'QUERY_POINT_DIMS': C, 'MEMORY_POINT_DIMS': C, 'REGRESSION': cfg}))
    with pytest.raises(ValueError, match='multiples of 128'):
        m.cuda().train()(d)


def test_train_then_eval(cuda):
    """after Adam steps the eval forward is the eval forward of a fresh model with the trained state (no stale weight cache)"""
    m = model('tf32')
    d = batch(2, seed=1)
    m.eval()
    with torch.no_grad():
        m(dict(d))
    m.train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    for _ in range(2):
        device_step(m, d)
        opt.step()
    m.eval()
    with torch.no_grad():
        got = m(dict(d))[0]['pred_boxes']
    fresh = model('tf32')
    fresh.load_state_dict(m.state_dict())
    fresh.eval()
    with torch.no_grad():
        want = fresh(dict(d))[0]['pred_boxes']
    assert torch.equal(got, want)


def test_peak_memory_below_autograd(cuda):
    d = batch(32, seed=7)
    m = model('tf32')
    device_step(m, d)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    device_step(m, d)
    ours = torch.cuda.max_memory_allocated() - base
    ref = model('tf32').reg
    del m
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    _autograd32(ref, d, True)
    theirs = torch.cuda.max_memory_allocated() - base
    print('B = 32 peak above the model: device step %.2f GB, float32 autograd %.2f GB' % (ours / 2**30, theirs / 2**30))
    assert ours < theirs

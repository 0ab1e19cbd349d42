"""CRM training on the device (detzero_b200/refine/train.py, csrc/refine_train.cu): one step against the reference's own float64
golden (tests/golden/crm_train.npz) and the float64 restatement (oracle/crm_train_ref.py), determinism, memory, train / eval
agreement, and each point pass against float64 at a shape with a partial last CTA wave."""
import os

import numpy as np
import pytest
import torch

from detzero_b200 import _lib, ops
from detzero_b200.config import AttrDict
from detzero_b200.refine.modules import RefineTemplate
from oracle import crm_train_ref, weights
from oracle import refine_inputs as ri

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'crm_train.npz')
SEED = 7301
# losses relative; running statistics norm-relative; point-encoder gradients norm-relative at B = 2 (golden) and B = 8 (restatement).
# A pooled row is an argmax over 256 rows: where the top two z of a (crop, channel) lie within rounding of each other, the device and
# float64 pick different rows and that pair's gradient flows through a different point.  In fp32 that happens about once per
# 1e6 pairs (none at B = 2, measured 8e-4 at B = 8's 8e5 pairs); in TF32 about once per 100 pairs (measured 0.09-0.13 on every
# point-encoder gradient).  Any fp32 or TF32 implementation, torch autograd with cuDNN TF32 included, differs from float64 the same
# way; the per-pass tests below check the arithmetic itself at tight bounds.
# Several gradients are 0 up to rounding: the bias of a BatchNorm whose output only reaches the loss through another conv + BatchNorm
# (pts_encoder_1.7, pts_encoder_2.1, pts_mlp.4) sums a gradient whose rows add up to 0.  Every gradient's scale is therefore floored
# at FLOOR times the largest point-encoder gradient.
FLOOR = 1e-2
# pts_encoder_2.1.bias sums the pooled gradient over the crops where the pooled output is positive; the per-box BatchNorm makes the
# pooled gradient add up to 0 over all crops, so what remains is the few crops whose pooled output is 0, and TF32 rounding moves
# it by 0.3-1.0 of its size: in TF32 it is not compared.
TOL = {'fp32': {'loss': 1e-5, 'stats': 1e-4, 'B2': 1e-4, 'B8': 1e-2},
       'tf32': {'loss': 5e-3, 'stats': 5e-3, 'B2': 0.25, 'B8': 0.25}}
SKIP = {'fp32': (), 'tf32': ('pts_encoder_2.1.bias',)}


def crm(mode, seed=SEED):
    cfg = ri.crm_cfg()
    cfg.COMPUTE_MODE = mode
    m = RefineTemplate(AttrDict({'NAME': 'ConfidenceRefineModel', 'QUERY_POINT_DIMS': 32, 'MEMORY_POINT_DIMS': 32, 'REGRESSION': cfg}))
    weights.load_seeded(m.reg, seed)                   # the reference module's keys (no 'reg.' prefix), as the golden seeds them
    return m.cuda().train()


def step(m, pts, iou):
    m.zero_grad(set_to_none=True)
    ret, tb, disp = m({'conf_points': pts, 'iou': iou})
    ret['loss'].backward()
    grads = {k: p.grad.detach().clone() for k, p in m.reg.named_parameters()}
    stats = {k[4:]: v.detach().clone() for k, v in m.state_dict().items()
             if k.endswith(('running_mean', 'running_var', 'num_batches_tracked'))}
    return ret, tb, disp, grads, stats


def err(got, ref, floor=0.0):
    got, ref = got.double().cpu(), ref.double().cpu()
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), floor)


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_matches_reference_golden(mode):
    gold = np.load(GOLD)
    tl, tg, ts = TOL[mode]['loss'], TOL[mode]['B2'], TOL[mode]['stats']
    m = crm(mode)
    pts = ri.crm_inputs(SEED, B=2)['conf_points'].cuda()
    iou = crm_train_ref.crm_train_iou(SEED, 2, pts.shape[1]).cuda()
    ret, tb, disp, grads, stats = step(m, pts, iou)
    assert set(ret) == {'loss'} and disp == {}
    assert set(tb) == {'bin_cls_loss', 'iou_loss', 'confidence_loss', 'full_loss'}
    for k in ('bin_cls_loss', 'iou_loss', 'confidence_loss'):
        assert abs(tb[k].item() - gold['loss.' + k]) <= tl * abs(gold['loss.' + k]), (k, tb[k].item(), gold['loss.' + k])
    assert tb['full_loss'].item() == tb['confidence_loss'].item()
    floor = FLOOR * max(np.abs(gold[k]).max() for k in gold.files if k.startswith('grad.'))
    errs = {}
    for k, g in grads.items():
        if 'grad.' + k in gold:
            errs[k] = err(g, torch.from_numpy(gold['grad.' + k]), floor)
        else:
            gsq = gold['gsq.' + k]
            p = crm_train_ref.probe(k, g.shape, SEED)
            scale = max(np.sqrt(gsq), floor * np.sqrt(g.numel()))
            errs[k] = max(abs((g.double() ** 2).sum().item() - gsq) / scale ** 2 / 2,
                          abs((g.double().cpu() * p).sum().item() - gold['gdot.' + k]) / (scale * p.norm().item()))
    bad = {k: e for k, e in errs.items() if e > tg and k not in SKIP[mode]}
    assert not bad, (bad, errs)
    for k, v in stats.items():
        if k.endswith('num_batches_tracked'):
            assert int(v) == 1, k
        else:
            assert err(v, torch.from_numpy(gold['bn.' + k])) <= ts, k


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_matches_restatement_mixed_box_num(mode):
    tl, tg, ts = TOL[mode]['loss'], TOL[mode]['B8'], TOL[mode]['stats']
    B, seed = 8, SEED + 1
    m = crm(mode, seed)
    sd = {k[4:]: v for k, v in m.state_dict().items() if k.startswith('reg.')}
    pts = ri.crm_inputs(seed, B=B)['conf_points'].cuda()
    iou = crm_train_ref.crm_train_iou(seed, B, pts.shape[1], box_num=[200, 1, 37, 100, 199, 150, 64, 12]).cuda()
    losses, rgrads, rstats = crm_train_ref.crm_train_step(sd, pts, iou, device='cuda')
    _, tb, _, grads, stats = step(m, pts, iou)
    for k, v in losses.items():
        assert abs(tb[k].item() - v) <= tl * abs(v), k
    floor = FLOOR * max(g.abs().max().item() for k, g in rgrads.items() if k.startswith('pts_encoder'))
    errs = {k: err(g, rgrads[k], floor) for k, g in grads.items()}
    bad = {k: e for k, e in errs.items() if e > tg and k not in SKIP[mode]}
    assert not bad, (bad, errs)
    for k, v in stats.items():
        if k.endswith('num_batches_tracked'):
            assert int(v) == int(rstats[k]) == 1, k
        else:
            assert err(v, rstats[k]) <= ts, k


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_is_deterministic(mode):
    pts = ri.crm_inputs(SEED, B=4)['conf_points'].cuda()
    iou = crm_train_ref.crm_train_iou(SEED, 4, pts.shape[1]).cuda()
    a, b = step(crm(mode), pts, iou), step(crm(mode), pts, iou)
    for k in a[1]:
        assert torch.equal(a[1][k], b[1][k]), k
    for i in (3, 4):
        for k in a[i]:
            assert torch.equal(a[i][k], b[i][k]), k


def test_step_memory():
    B = 16
    pts = ri.crm_inputs(SEED, B=B)['conf_points'].cuda()
    iou = crm_train_ref.crm_train_iou(SEED, B, pts.shape[1]).cuda()
    m = crm('tf32')
    step(m, pts, iou)                                   # workspaces and caches at this shape
    torch.cuda.synchronize()
    m.zero_grad(set_to_none=True)
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step(m, pts, iou)
    torch.cuda.synchronize()
    rise = torch.cuda.max_memory_allocated() - base
    assert rise < 4 * pts.numel() * 4 + (512 << 20), rise


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_training_then_eval_agree(mode):
    B = 4
    pts = ri.crm_inputs(SEED + 2, B=B)['conf_points'].cuda()
    iou = crm_train_ref.crm_train_iou(SEED + 2, B, pts.shape[1]).cuda()
    pts[..., 0] += 2 * iou[..., None].clamp(0, 1)      # a learnable signal: the first feature shifts with the label
    m = crm(mode)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    losses = []
    for _ in range(6):
        opt.zero_grad(set_to_none=True)
        ret, tb, _ = m({'conf_points': pts, 'iou': iou})
        ret['loss'].backward()
        opt.step()
        m.update_global_step()
        losses.append(ret['loss'].item())
    assert losses[-1] < losses[0], losses
    assert int(m.global_step) == 6
    m.eval()
    got = m({'conf_points': pts})[0]['pred_score']
    fresh = crm(mode).eval()
    fresh.load_state_dict(m.state_dict())
    ref = fresh({'conf_points': pts})[0]['pred_score']
    assert torch.equal(got, ref)


# ---- each pass against float64 --------------------------------------------------------------------------------------------
def _pass_ref(x, W, tab, shift4, sel, dsel, P):
    """float64 statement of dz_crm_point_pass: {pass: (stats u, stats v)}, extremes, dW"""
    d = lambda t: t.double()                                                    # noqa: E731
    x, (W1, W2, W3, W4p) = d(x), [d(w) for w in W]
    t = d(tab)
    R = x.shape[0]
    crops = R // P
    rows = torch.arange(R, device=x.device)
    lay = lambda l, z, C: (t[l, 0, :C] * z + t[l, 1, :C]).clamp_min(0)        # noqa: E731
    xh = lambda l, z, C: (z - t[l, 2, :C]) * t[l, 3, :C]                      # noqa: E731
    z1 = x @ W1.t(); y1 = lay(0, z1, 128)
    z2 = y1 @ W2.t(); y2 = lay(1, z2, 128)
    z3 = y2 @ W3.t()
    z4 = y2 @ W4p.t() + d(shift4).repeat_interleave(P, 0)
    out = {p: (z.sum(0), (z * z).sum(0)) for p, z in ((1, z1), (2, z2), (3, z3), (4, z4))}
    dz = []
    for l, z in ((2, z3), (3, z4)):
        s, dd = sel[l - 2].long(), d(dsel[l - 2])
        dh = torch.zeros_like(z)
        hit = (rows % P)[:, None] == s.repeat_interleave(P, 0)
        dh[hit] = dd.repeat_interleave(P, 0)[hit]
        dz.append(t[l, 0] * (dh - t[l, 4] - xh(l, z, 256) * t[l, 5]))
    dz3, dz4 = dz
    dy2 = dz4 @ W4p + dz3 @ W3
    dh2 = dy2 * ((t[1, 0, :128] * z2 + t[1, 1, :128]) > 0)
    out[5] = (dh2.sum(0), (dh2 * xh(1, z2, 128)).sum(0))
    dz2 = t[1, 0, :128] * (dh2 - t[1, 4, :128] - xh(1, z2, 128) * t[1, 5, :128])
    dy1 = dz2 @ W2
    dh1 = dy1 * ((t[0, 0, :128] * z1 + t[0, 1, :128]) > 0)
    out[6] = (dh1.sum(0), (dh1 * xh(0, z1, 128)).sum(0))
    dz1 = t[0, 0, :128] * (dh1 - t[0, 4, :128] - xh(0, z1, 128) * t[0, 5, :128])
    dW = {5: torch.cat([dz4.t() @ y2, dz3.t() @ y2]).reshape(-1), 6: (dz2.t() @ y1).reshape(-1), 7: (dz1.t() @ x).reshape(-1)}
    return out, {3: z3.view(crops, P, -1), 4: z4.view(crops, P, -1)}, dW


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_point_passes_against_float64(mode):
    torch.manual_seed(5)
    crops, P, c0 = 150, 128, 32                         # 150 crops on a 132-CTA grid: a partial last wave
    dev = 'cuda'
    x = torch.randn(crops * P, c0, device=dev)
    W = [torch.randn(n, k, device=dev) / k ** 0.5 for n, k in ((128, c0), (128, 128), (256, 128), (256, 128))]
    tab = torch.zeros(4, 6, 256, device=dev)
    tab[:, 0] = torch.rand(4, 256, device=dev) + 0.5
    tab[:, 0, :64] *= -1                                # negative BN scales pool at the min row
    tab[:, 1] = torch.randn(4, 256, device=dev) * 0.3
    tab[:, 2] = torch.randn(4, 256, device=dev) * 0.1
    tab[:, 3] = torch.rand(4, 256, device=dev) + 0.5
    tab[:, 4:] = torch.randn(4, 2, 256, device=dev) * 1e-3
    shift4 = torch.randn(crops, 256, device=dev)
    sel = torch.randint(0, P, (2, crops, 256), device=dev, dtype=torch.int32)
    dsel = torch.randn(2, crops, 256, device=dev)
    wf = tuple(w.t().contiguous() for w in W)
    wb = (W[1].contiguous(), W[2].contiguous(), W[3].contiguous())
    ref, zref, dref = _pass_ref(x, W, tab, shift4, sel, dsel, P)
    # backward passes: a ReLU mask taken at a z within rounding of its threshold flips a whole dh element, so they get more room,
    # pass 7 (dW1, behind two masks) the most
    tol_f, tol_b = (1e-5, 1e-4) if mode == 'fp32' else (5e-3, 2e-2)
    tol_7 = 5e-4 if mode == 'fp32' else 5e-2
    m = _lib.MODES[mode]
    for p in range(1, 8):
        stats = torch.empty(512, dtype=torch.float64, device=dev)
        zext = torch.empty(2, crops, 256, device=dev)
        iext = torch.empty(2, crops, 256, dtype=torch.int32, device=dev)
        csum = torch.empty(crops, 256, dtype=torch.float64, device=dev)
        slab = torch.empty(2 * 256 * 128, dtype=torch.float64, device=dev) if p >= 5 else None
        ops.crm_point_pass(p, m, x, P, wf, wb, tab, shift4, sel, dsel, zext, iext, csum, stats, slab)
        tol = tol_f if p <= 4 else tol_b if p < 7 else tol_7
        if p <= 6:
            C = 256 if p in (3, 4) else 128
            assert err(stats[:C], ref[p][0]) <= tol and err(stats[256:256 + C], ref[p][1]) <= tol, p
        if p in (3, 4):
            z = zref[p]
            zmax, zmin = z.max(1)[0], z.min(1)[0]
            spread = (zmax - zmin).abs().max().item()
            assert err(zext[0], zmax) <= tol and err(zext[1], zmin) <= tol, p
            # the chosen rows hold the extreme value (up to the compute mode) and, among exact float64 ties, the lowest row
            at_max = z.gather(1, iext[0].long().unsqueeze(1)).squeeze(1)
            at_min = z.gather(1, iext[1].long().unsqueeze(1)).squeeze(1)
            assert (at_max - zmax).abs().max().item() <= tol * spread and (at_min - zmin).abs().max().item() <= tol * spread, p
            if p == 4:
                assert err(csum, z.sum(1)) <= tol
        if p >= 5:
            n = dref[p].numel()
            assert err(slab[:n], dref[p]) <= tol, p

"""CRM training on the device (detzero_b200/refine/train.py, csrc/refine_train.cu): one step against the reference's own float64
golden (tests/golden/crm_train.npz) and the float64 restatement (oracle/crm_train_ref.py), determinism, memory, train / eval
agreement, each point pass against float64 (exact arithmetic bit for bit, random data at derived per-element bounds, the ties a
padded box makes), the steps pooled at the device's rows, and what the train-mode point encoders refuse."""
import os

import numpy as np
import pytest
import torch

from detzero_b200 import _lib, ops, synthetic
from detzero_b200.config import AttrDict
from detzero_b200.refine import data as rdata, train
from detzero_b200.refine.modules import RefineTemplate
from oracle import crm_train_ref, weights
from oracle import refine_inputs as ri

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'crm_train.npz')
SEED = 7301
U32 = 2.0 ** -24            # fp32 unit roundoff
U_TF32 = 2.0 ** -11         # an operand rounded to nearest TF32 (10 explicit mantissa bits)
TM = 64                     # rows per tile of the point passes
# Step tolerances.  fp32: 1e-5 relative on losses, 1e-4 norm-relative (max |error| / max |reference|) on gradients and running
# statistics.  tf32: every point-layer GEMM rounds both operands to TF32, a relative error up to 2 * 2^-11 per product; independent
# roundings over a reduction of length K grow like sqrt(K) and are damped by the same 1/sqrt(K) of a BatchNorm-normalised output, so
# each layer adds about 2 * 2^-11 = 1e-3 relative.  The forward chains the four point layers and their BatchNorm statistics (4e-3:
# 5e-3 on the losses, the running statistics and the pooled output); the backward chains the same four again (8e-3: 1e-2 on the
# gradients).  The per-box layers run through torch autograd in fp32 in both modes.
TOL = {'fp32': {'loss': 1e-5, 'grad': 1e-4, 'stats': 1e-4},
       'tf32': {'loss': 5e-3, 'grad': 1e-2, 'stats': 5e-3}}
# A bound looser than these, with its cause: BatchNorm backwards make dZ of every layer sum to 0 over its rows (the point layers over
# B*L*P rows, the per-box layers over B*L boxes), and a bias whose output reaches the loss through another conv + BatchNorm sums such
# a remainder, so several gradients are small remainders of large terms that keep the rounding of the large ones.  Plain float32
# autograd of the same forward (the restatement run in float32 at the same pooled rows, TF32 matmuls in the tf32 mode) has the same
# conditioning; a gradient is allowed ASSOC times the error that autograd makes on it, when that is larger than the bound above.
# This is what the fp32 per-box (pts_mlp) gradients at B = 8 on Gaussian points are: pooled at the device's rows, pts_mlp.0.weight is
# 4.7e-3 off float64 and float32 autograd 4.4e-3, while the pooled output they take is within 3.7e-6 of float64 (measured on an H100
# 80GB HBM3 at 700 W).  ASSOC is measured, not derived: the largest ratio seen was 3.1, on pts_mlp.4.weight in fp32 at B = 8; 8
# leaves room for a different batch.
ASSOC = 8
# BatchNorm biases whose output reaches the loss only through another conv + BatchNorm sum a gradient whose rows add up to 0: their
# gradient is 0 up to rounding, so every gradient's scale is floored at FLOOR times the largest gradient.
FLOOR = 1e-2


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


def clone_sd(m):
    return {k[4:]: v.detach().clone() for k, v in m.state_dict().items() if k.startswith('reg.')}


def check_stats(stats, ref, tol):
    for k, v in stats.items():
        if k.endswith('num_batches_tracked'):
            assert int(v) == int(ref[k]) == 1, k
        else:
            assert err(v, ref[k]) <= tol, (k, err(v, ref[k]))


def ref32(sd, pts, iou, mode, **kw):
    """plain float32 (tf32: TF32 matmul) autograd of the restatement"""
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = mode == 'tf32'
    try:
        return crm_train_ref.crm_train_step(sd, pts, iou, device='cuda', dtype=torch.float32, **kw)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def check_grads(grads, ref_err, ag, tol):
    """each gradient within the larger of tol and ASSOC times the error float32 autograd makes on it (ag)"""
    errs = {k: ref_err(k, g) for k, g in grads.items()}
    bad = {k: (e, ag[k]) for k, e in errs.items() if e > max(tol, ASSOC * ag[k])}
    assert not bad, bad


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_matches_reference_golden(mode):
    gold = np.load(GOLD)
    tol = TOL[mode]
    m = crm(mode)
    sd = clone_sd(m)
    pts = ri.crm_inputs(SEED, B=2)['conf_points'].cuda()
    iou = crm_train_ref.crm_train_iou(SEED, 2, pts.shape[1]).cuda()
    ret, tb, disp, grads, stats = step(m, pts, iou)
    assert set(ret) == {'loss'} and disp == {}
    assert set(tb) == {'bin_cls_loss', 'iou_loss', 'confidence_loss', 'full_loss'}
    for k in ('bin_cls_loss', 'iou_loss', 'confidence_loss'):
        assert abs(tb[k].item() - gold['loss.' + k]) <= tol['loss'] * abs(gold['loss.' + k]), (k, tb[k].item(), gold['loss.' + k])
    assert tb['full_loss'].item() == tb['confidence_loss'].item()
    floor = FLOOR * max(np.abs(gold[k]).max() for k in gold.files if k.startswith('grad.'))

    def gerr(k, g):
        if 'grad.' + k in gold:
            return err(g, torch.from_numpy(gold['grad.' + k]), floor)
        gsq = gold['gsq.' + k]
        p = crm_train_ref.probe(k, g.shape, SEED)
        scale = max(np.sqrt(gsq), floor * np.sqrt(g.numel()))
        return max(abs((g.double() ** 2).sum().item() - gsq) / scale ** 2 / 2,
                   abs((g.double().cpu() * p).sum().item() - gold['gdot.' + k]) / (scale * p.norm().item()))

    _, g32, _ = ref32(sd, pts, iou, mode)             # float32 autograd pools at its own argmax, as the golden does
    check_grads(grads, gerr, {k: gerr(k, g) for k, g in g32.items()}, tol['grad'])
    check_stats(stats, {k[3:]: torch.from_numpy(gold[k]) for k in gold.files if k.startswith('bn.')}, tol['stats'])


def device_step_at_rows(mode, seed, pts, iou):
    """one device step, the device's pooled output (a second module with the same weights: the step itself does not return it) and
    the float64 restatement pooled at the device's rows"""
    m = crm(mode, seed)
    sd = clone_sd(m)
    _, tb, _, grads, stats = step(m, pts, iou)
    rows = {k: v.cpu() for k, v in m.reg.pooled_rows.items()}
    with torch.no_grad():
        m2 = crm(mode, seed)
        pool = train.point_encoders(m2.reg, pts)
    for k in rows:
        assert torch.equal(m2.reg.pooled_rows[k].cpu(), rows[k]), k
    rec = {}
    losses, rgrads, rstats = crm_train_ref.crm_train_step(sd, pts, iou, device='cuda', pooled_rows=rows, record=rec)
    return sd, rows, tb, grads, stats, pool, losses, rgrads, rstats, rec


def check_at_rows(mode, seed, pts, iou):
    tol = TOL[mode]
    sd, rows, tb, grads, stats, pool, losses, rgrads, rstats, rec = device_step_at_rows(mode, seed, pts, iou)
    for k, v in losses.items():
        assert abs(tb[k].item() - v) <= tol['loss'] * abs(v), (k, tb[k].item(), v)
    # the pooled output itself, element by element, each channel against its largest value over the crops; allowed ASSOC times the
    # error of float32 autograd at the same rows where that is larger.  The tf32 bound above assumes BatchNorm-normalised operands;
    # the first layer rounds the raw point features to TF32, and the built inputs hold features far from zero mean (coordinates,
    # the box's size), whose rounding float32 autograd with TF32 matmuls shares
    ref = rec['pool']
    scale = ref.abs().amax(dim=0, keepdim=True).clamp_min(1e-30)
    rel = lambda t: ((t.double() - ref).abs() / scale).max().item()          # noqa: E731
    rec32 = {}
    _, g32, _ = ref32(sd, pts, iou, mode, pooled_rows=rows, record=rec32)
    perr, perr32 = rel(pool), rel(rec32['pool'])
    assert perr <= max(tol['stats'], ASSOC * perr32), (perr, perr32)
    floor = FLOOR * max(g.abs().max().item() for g in rgrads.values())
    ref_err = lambda k, g: err(g, rgrads[k], floor)                  # noqa: E731
    check_grads(grads, ref_err, {k: ref_err(k, g) for k, g in g32.items()}, tol['grad'])
    check_stats(stats, rstats, tol['stats'])


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_matches_restatement_at_device_pooled_rows(mode):
    """B = 8, mixed box_num, against the float64 restatement pooled at the rows the device picked: arithmetic, without argmax flips"""
    B, seed = 8, SEED + 1
    pts = ri.crm_inputs(seed, B=B)['conf_points'].cuda()
    iou = crm_train_ref.crm_train_iou(seed, B, pts.shape[1], box_num=[200, 1, 37, 100, 199, 150, 64, 12]).cuda()
    check_at_rows(mode, seed, pts, iou)


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_pooled_rows_against_float64(mode):
    """B = 8: every row the device pools at holds, in float64, a value within the forward bound of the float64 maximum of its crop
    (the pooled value is the ReLU output: the max row of z where a >= 0, the min row where a < 0), and the device pools at a row
    whose value is below the maximum no more often than plain float32 (tf32: TF32) autograd does"""
    B, seed = 8, SEED + 1
    m = crm(mode, seed)
    sd = clone_sd(m)
    pts = ri.crm_inputs(seed, B=B)['conf_points'].cuda()
    iou = crm_train_ref.crm_train_iou(seed, B, pts.shape[1]).cuda()
    step(m, pts, iou)
    rec64, rec32 = {}, {}
    crm_train_ref.crm_train_step(sd, pts, iou, device='cuda', record=rec64)
    ref32(sd, pts, iou, mode, record=rec32)
    for k in ('enc1', 'enc2'):
        y = rec64[k]                                                  # (crops, P, 256) float64 inputs of the max
        dev = m.reg.pooled_rows[k].long()
        top = y.max(dim=1)[0]
        at = y.gather(1, dev.unsqueeze(1)).squeeze(1)
        bound = 2 * TOL[mode]['stats'] * y.abs().amax(dim=1)
        assert ((top - at) <= bound).all(), (k, ((top - at) / bound.clamp_min(1e-30)).max().item())
        # a flip: the chosen row's float64 value is below the maximum (ties, ReLU zeros included, are not flips)
        at32 = y.gather(1, rec32[k].max(dim=1)[1].unsqueeze(1)).squeeze(1)
        flips_dev, flips_ag = int((at < top).sum()), int((at32 < top).sum())
        assert flips_dev <= 2 * flips_ag + 2, (k, flips_dev, flips_ag, top.numel())


def production_inputs(B=8, L=200):
    """conf_points built on the device from a tracked synthetic sequence: boxes with no point (their crops are all one encoded zero
    point), with a few points and with more than 256 (sampled), and tracks shorter than L"""
    s = synthetic.synthetic_sequence(SEED, frames=L, tracks=B, L=L, n_background=2000, lengths=[200, 150, 37, 1, 90, 12, 199, 64])
    dev = torch.device('cuda')
    tb = rdata.TrackBatch(s['boxes'], s['frame_of_box'], s['scores'], s['box_num'], s['cls'], s['track_uid'], dev)
    out = rdata.confidence_inputs(torch.from_numpy(s['frames']).to(dev), s['frame_offsets'], torch.from_numpy(s['poses']).to(dev), tb,
                                  seed=SEED, return_selection=True)
    counts = out['crop_counts'].cpu()
    box_num = torch.from_numpy(np.asarray(s['box_num']))
    live = torch.arange(L)[None] < box_num[:, None]
    c = counts[live]
    assert (c == 0).any() and ((c > 0) & (c < 64)).any() and (c > 256).any(), c
    assert (box_num < L).sum() >= B - 2
    iou = crm_train_ref.crm_train_iou(SEED, B, L, box_num=box_num.tolist())
    return out['conf_points'].float().contiguous(), iou.cuda()


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_on_production_inputs_at_device_pooled_rows(mode):
    """the only step whose crops hold the padded-sample ties: the device's pooled rows, gradients and pooled output against the float64
    restatement at those rows"""
    pts, iou = production_inputs()
    check_at_rows(mode, SEED + 5, pts, iou)


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
# A GEMM output's element bound: |z - z64| <= (c + (K + 2) u) S, S = sum |a| |b| over the reduction, u = 2^-24 for the fp32
# accumulation over K terms, c = 0 in fp32 and 2 * 2^-11 in tf32 (both operands rounded to nearest TF32).  An operand that carries an
# error bound e of its own adds |e| |b| summed over the reduction.  The weight gradients accumulate each 64-row tile in fp32 and the
# tiles in float64: K = 64.
def gamma(mode, K):
    return (0.0 if mode == 'fp32' else 2 * U_TF32) + (K + 2) * U32


# The bound above is the worst case: every term's rounding of the same sign.  Roundings to nearest are nearly independent, so the
# root mean square of a GEMM output's error over all elements is held as well to the sum in quadrature, S2 = sum (a b)^2 over the
# reduction, plus the root mean square of what its operands' bounds carry in: (c + 2 sqrt(K) 2^-24) sqrt(mean S2) + rms(carried).
def rms_ok(diff, S2, carried, mode, K):
    c = (0.0 if mode == 'fp32' else 2 * U_TF32) + 2 * K ** 0.5 * U32
    rms = lambda t: t.double().pow(2).mean().sqrt().item()                   # noqa: E731
    return rms(diff) <= c * S2.mean().sqrt().item() + rms(carried)


def _pass_ref(x, W, tab, shift4, sel, dsel, P, mode):
    """float64 statement of dz_crm_point_pass, with the rounding bound of every output.  Returns {name: (value, element bound, S2 |
    None, carried | None)} for the statistics 'u1'..'v6', the z of the pooled layers 'z3', 'z4' (crops, P, 256), 'csum', and the weight
    gradients 'w5', 'w6', 'w7' (flattened as the slab); and the ReLU pre-activations of layers 1 and 2 with the bound of each."""
    d = lambda t: t.double()                                                    # noqa: E731
    x, (W1, W2, W3, W4p) = d(x), [d(w) for w in W]
    t = d(tab)
    R, c0 = x.shape
    crops = R // P
    A = lambda t_: t_.abs()                                                      # noqa: E731
    DS = R * 2.0 ** -53                          # a float64 sum over the rows
    out = {}
    formed = []                                  # elementwise values the kernel forms, for the exact test's premises

    def gemm(a, ea, w, K):                       # a (R, K) with bound ea, times w^T (w (N, K)): value, bound
        return a @ w.t(), gamma(mode, K) * ((A(a) + ea) @ A(w).t()) + ea @ A(w).t()

    def act(l, z, ez, C):                        # ReLU(fma(a, z, b)): value, bound, pre-activation, its margin bound
        a, b = t[l, 0, :C], t[l, 1, :C]
        pre = a * z + b
        formed.append(pre)
        return pre.clamp_min(0), A(a) * ez + U32 * (A(pre) + A(a) * ez), pre, A(a) * ez

    def stats(p, z, ez):
        out['u%d' % p] = (z.sum(0), ez.sum(0) + DS * A(z).sum(0), None, None)
        out['v%d' % p] = ((z * z).sum(0), (ez * (2 * A(z) + ez)).sum(0) + DS * (z * z).sum(0), None, None)

    zero = torch.zeros_like(x)
    z1, e1 = gemm(x, zero, W1, c0)
    y1, ey1, pre1, m1 = act(0, z1, e1, 128)
    z2, e2 = gemm(y1, ey1, W2, 128)
    y2, ey2, pre2, m2 = act(1, z2, e2, 128)
    z3, e3 = gemm(y2, ey2, W3, 128)
    z4, g4 = gemm(y2, ey2, W4p, 128)
    formed.append(z4)
    sh = d(shift4).repeat_interleave(P, 0)
    z4 = z4 + sh
    e4 = g4 + U32 * (A(z4) + g4)
    for p, z, e in ((1, z1, e1), (2, z2, e2), (3, z3, e3), (4, z4, e4)):
        stats(p, z, e)
    out['z3'] = (z3.view(crops, P, -1), e3.view(crops, P, -1), None, None)
    out['z4'] = (z4.view(crops, P, -1), e4.view(crops, P, -1), None, None)
    out['csum'] = (z4.view(crops, P, -1).sum(1), e4.view(crops, P, -1).sum(1) + DS * A(z4).view(crops, P, -1).sum(1), None, None)

    def dz(l, z, ez, dh, edh, C):                # a (dh - m1 - xhat m2), xhat = (z - mean) rstd: value, bound, xhat, its bound
        a, mu, rs, k1, k2 = (t[l, i, :C] for i in (0, 2, 3, 4, 5))
        xh = (z - mu) * rs
        exh = A(rs) * ez * (1 + U32) + 3 * U32 * (A(xh) + A(rs) * ez)
        v = a * (dh - k1 - xh * k2)
        formed.extend([z - mu, xh, dh - k1, xh * k2, dh - k1 - xh * k2, v])
        return v, A(a) * (edh + A(k2) * exh) + 4 * U32 * A(a) * (A(dh) + edh + A(k1) + A(k2) * (A(xh) + exh)), xh, exh

    def wgrad(name, dzv, edz, y, ey):            # sum over rows of dz^T y, 64-row tiles in fp32
        S = (A(dzv) + edz).t() @ (A(y) + ey)
        carried = edz.t() @ (A(y) + ey) + A(dzv).t() @ ey
        return dzv.t() @ y, gamma(mode, TM) * S + carried, dzv.pow(2).t() @ y.pow(2), carried

    rows = torch.arange(R, device=x.device)
    dzs = []
    for l, z, ez in ((2, z3, e3), (3, z4, e4)):
        s, dd = sel[l - 2].long(), d(dsel[l - 2])
        dh = torch.zeros_like(z)
        hit = (rows % P)[:, None] == s.repeat_interleave(P, 0)
        dh[hit] = dd.repeat_interleave(P, 0)[hit]
        dzs.append(dz(l, z, ez, dh, torch.zeros_like(z), 256)[:2])
    (dz3, edz3), (dz4, edz4) = dzs
    parts = [wgrad('w4p', dz4, edz4, y2, ey2), wgrad('w3', dz3, edz3, y2, ey2)]
    out['w5'] = tuple(torch.cat([q[i].reshape(-1) for q in parts]) for i in range(4))
    dy2 = dz4 @ W4p + dz3 @ W3
    edy2 = gamma(mode, 256) * ((A(dz4) + edz4) @ A(W4p) + (A(dz3) + edz3) @ A(W3)) + edz4 @ A(W4p) + edz3 @ A(W3)
    k2 = (pre2 > 0).double()
    dh2, edh2 = dy2 * k2, edy2 * k2
    dz2, edz2, xh2, exh2 = dz(1, z2, e2, dh2, edh2, 128)
    out['u5'] = (dh2.sum(0), edh2.sum(0) + DS * A(dh2).sum(0), None, None)
    out['v5'] = ((dh2 * xh2).sum(0), (edh2 * (A(xh2) + exh2) + A(dh2) * exh2).sum(0) + DS * A(dh2 * xh2).sum(0), None, None)
    out['w6'] = tuple(q.reshape(-1) for q in wgrad('w2', dz2, edz2, y1, ey1))
    dy1 = dz2 @ W2
    edy1 = gamma(mode, 128) * ((A(dz2) + edz2) @ A(W2)) + edz2 @ A(W2)
    k1 = (pre1 > 0).double()
    dh1, edh1 = dy1 * k1, edy1 * k1
    dz1, edz1, xh1, exh1 = dz(0, z1, e1, dh1, edh1, 128)
    out['u6'] = (dh1.sum(0), edh1.sum(0) + DS * A(dh1).sum(0), None, None)
    out['v6'] = ((dh1 * xh1).sum(0), (edh1 * (A(xh1) + exh1) + A(dh1) * exh1).sum(0) + DS * A(dh1 * xh1).sum(0), None, None)
    out['w7'] = tuple(q.reshape(-1) for q in wgrad('w1', dz1, edz1, x, zero))
    inter = {'x': x, 'z1': z1, 'y1': y1, 'z2': z2, 'y2': y2, 'z3': z3, 'z4': z4, 'dz3': dz3, 'dz4': dz4, 'dy2': dy2, 'dh2': dh2,
             'xh2': xh2, 'dz2': dz2, 'dy1': dy1, 'dh1': dh1, 'xh1': xh1, 'dz1': dz1}
    inter.update(('formed%d' % i, v) for i, v in enumerate(formed))
    return out, ((pre1, m1), (pre2, m2)), inter


def run_passes(mode, x, P, W, tab, shift4, sel, dsel):
    """every pass on the device: {name: value} with the names of _pass_ref, plus 'i3', 'i4' the extreme rows and 'x3', 'x4' the
    extreme z, each (2, crops, 256) [max, min]"""
    dev = x.device
    crops = x.shape[0] // P
    wf = tuple(w.t().contiguous() for w in W)
    wb = (W[1].contiguous(), W[2].contiguous(), W[3].contiguous())
    got = {}
    for p in range(1, 8):
        stats = torch.full((512,), float('nan'), dtype=torch.float64, device=dev)
        zext = torch.full((2, crops, 256), float('nan'), device=dev)
        iext = torch.full((2, crops, 256), -1, dtype=torch.int32, device=dev)
        csum = torch.full((crops, 256), float('nan'), dtype=torch.float64, device=dev)
        slab = torch.full((2 * 256 * 128,), float('nan'), dtype=torch.float64, device=dev) if p >= 5 else None
        ops.crm_point_pass(p, _lib.MODES[mode], x, P, wf, wb, tab, shift4, sel, dsel, zext, iext, csum, stats, slab)
        if p <= 6:
            C = 256 if p in (3, 4) else 128
            got['u%d' % p], got['v%d' % p] = stats[:C], stats[256:256 + C]
        if p in (3, 4):
            got['x%d' % p], got['i%d' % p] = zext, iext
        if p == 4:
            got['csum'] = csum
        if p >= 5:
            n = {5: 2 * 256 * 128, 6: 128 * 128, 7: 128 * x.shape[1]}[p]
            got['w%d' % p] = slab[:n]
    return got


def lowest_extreme_rows(z):
    """per (crop, channel) of z (crops, P, C): the max and min and the lowest row holding each"""
    P = z.shape[1]
    r = torch.arange(P, device=z.device).view(1, P, 1)
    out = []
    for v in (z.max(1)[0], z.min(1)[0]):
        out.append((v, torch.where(z == v.unsqueeze(1), r, P).min(1)[0]))
    return out


def check_against_bounds(mode, got, ref):
    """every output within its element bound, the weight gradients within their RMS bound too; the extreme rows: the chosen row is
    the lowest of the float64 tie set wherever no other row lies within the bounds, and its value within the bounds elsewhere"""
    for k, (v, bound, S2, carried) in ref.items():
        if k in ('z3', 'z4'):
            continue
        diff = (got[k].double() - v).abs()
        assert (diff <= bound).all(), (k, (diff / bound.clamp_min(1e-300)).max().item())
        if S2 is not None:
            assert rms_ok(diff, S2, carried, mode, TM), k
    clear_at = {}
    for p in (3, 4):
        z, ez = ref['z%d' % p][:2]
        for h, (v, lo) in enumerate(lowest_extreme_rows(z)):
            idx = got['i%d' % p][h].long()
            assert (idx >= 0).all() and (idx < z.shape[1]).all(), p
            at = z.gather(1, idx.unsqueeze(1)).squeeze(1)
            eat = ez.gather(1, idx.unsqueeze(1)).squeeze(1)
            # the device's extreme is the z it computed at that row
            assert ((got['x%d' % p][h].double() - at).abs() <= eat).all(), (p, h)
            # ... which lies within both rows' bounds of the float64 extreme
            elo = ez.gather(1, lo.unsqueeze(1)).squeeze(1)
            assert ((at - v).abs() <= eat + elo).all(), (p, h)
            # where no row outside the float64 tie set comes within the bounds, the chosen row is the tie set's lowest
            sgn = 1 if h == 0 else -1
            near = (sgn * (v.unsqueeze(1) - z) <= ez + ez.max(1, keepdim=True)[0]) & (z != v.unsqueeze(1))
            clear = ~near.any(1)
            assert torch.equal(idx[clear], lo[clear]), (p, h, int((idx != lo)[clear].sum()))
            clear_at[p, h] = clear
    return clear_at


FORWARD = ('u1', 'v1', 'u2', 'v2', 'u3', 'v3', 'u4', 'v4', 'csum', 'z3', 'z4')


def random_tab(gen, dev):
    tab = torch.zeros(4, 6, 256, device=dev)
    tab[:, 0] = torch.rand(4, 256, generator=gen, device=dev) + 0.5
    tab[:, 0, :64] *= -1                                # negative BN scales pool at the min row
    tab[:, 1] = torch.randn(4, 256, generator=gen, device=dev) * 0.3
    tab[:, 2] = torch.randn(4, 256, generator=gen, device=dev) * 0.1
    tab[:, 3] = torch.rand(4, 256, generator=gen, device=dev) + 0.5
    tab[:, 4:] = torch.randn(4, 2, 256, generator=gen, device=dev) * 1e-2
    return tab


def clear_rows(mode, n, c0, W, tab, gen, dev):
    """n Gaussian point rows none of whose ReLU masks (layers 1 and 2, the ones the backward passes apply) lies within its rounding
    bound of the threshold: rows are independent through the 1x1 layers, so a row with an ambiguous mask is drawn again"""
    keep = []
    have = 0
    while have < n:
        x = torch.randn(2 * (n - have) + 64, c0, generator=gen, device=dev)
        d = lambda t: t.double()                                                    # noqa: E731
        W1, W2 = d(W[0]), d(W[1])
        t = d(tab)
        z1 = d(x) @ W1.t()
        e1 = gamma(mode, c0) * (d(x).abs() @ W1.abs().t())
        pre1 = t[0, 0, :128] * z1 + t[0, 1, :128]
        y1 = pre1.clamp_min(0)
        ey1 = t[0, 0, :128].abs() * e1 + U32 * (pre1.abs() + t[0, 0, :128].abs() * e1)
        z2 = y1 @ W2.t()
        e2 = gamma(mode, 128) * ((y1 + ey1) @ W2.abs().t()) + ey1 @ W2.abs().t()
        pre2 = t[1, 0, :128] * z2 + t[1, 1, :128]
        ok = ((pre1.abs() > t[0, 0, :128].abs() * e1).all(1) & (pre2.abs() > t[1, 0, :128].abs() * e2).all(1))
        keep.append(x[ok])
        have += int(ok.sum())
    return torch.cat(keep)[:n].contiguous()


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
@pytest.mark.parametrize('crops,P,c0', [(1, 64, 8), (133, 256, 32), (264, 64, 64), (150, 512, 32)])
def test_point_passes_against_float64(mode, crops, P, c0):
    """random data at per-element bounds derived from float64 sums of magnitudes: one crop of one tile; the production P and c0 on
    one crop more than the 132-CTA grid; two crops per CTA at the largest c0; eight tiles per crop on a partial last wave"""
    dev = 'cuda'
    gen = torch.Generator(device=dev).manual_seed(1000 * crops + P + c0)
    W = [torch.randn(n, k, generator=gen, device=dev) / k ** 0.5 for n, k in ((128, c0), (128, 128), (256, 128), (256, 128))]
    tab = random_tab(gen, dev)
    x = clear_rows(mode, crops * P, c0, W, tab, gen, dev)
    shift4 = torch.randn(crops, 256, generator=gen, device=dev)
    sel = torch.randint(0, P, (2, crops, 256), generator=gen, device=dev, dtype=torch.int32)
    dsel = torch.randn(2, crops, 256, generator=gen, device=dev)
    ref, masks, _ = _pass_ref(x, W, tab, shift4, sel, dsel, P, mode)
    for pre, m in masks:                                # the premise of the tight backward bounds: no ambiguous ReLU mask
        assert (pre.abs() > m).all()
    check_against_bounds(mode, run_passes(mode, x, P, W, tab, shift4, sel, dsel), ref)


# ---- exact arithmetic: every value the kernel forms is representable, so fp32 and TF32 must both give float64's bits ---------------
def tf32_round(t):
    """round to nearest TF32 (10 explicit mantissa bits), ties away from zero, as cvt.rna.tf32.f32"""
    m, e = torch.frexp(t.double())
    return torch.ldexp(torch.sign(m) * torch.floor(m.abs() * 2 ** 11 + 0.5) / 2 ** 11, e)


def grid(t):
    """the coarsest power of two every nonzero element of t is an integer multiple of"""
    t = t.double()
    t = t[t != 0]
    k = 40
    while k > -60 and not torch.equal(t * 2.0 ** -k, torch.round(t * 2.0 ** -k)):
        k -= 1
    return 2.0 ** k


def exact_inputs(crops, P, c0, dev):
    g = torch.Generator(device='cpu').manual_seed(77)
    ri_ = lambda lo, hi, shape: torch.randint(lo, hi, shape, generator=g).float()       # noqa: E731

    def sparse_w(n, k, per):                              # per nonzeros of +-1 in each output row
        w = torch.zeros(n, k)
        for i in range(n):
            j = torch.randperm(k, generator=g)[:per]
            w[i, j] = ri_(0, 2, (per,)) * 2 - 1
        return w

    x = ri_(-1, 2, (crops * P, c0))
    W = [sparse_w(128, c0, 4), sparse_w(128, 128, 3), sparse_w(256, 128, 2), sparse_w(256, 128, 2)]
    tab = torch.zeros(4, 6, 256)
    tab[:, 0] = 2.0 ** ri_(-1, 1, (4, 256))                # a: powers of two ...
    tab[:, 0] *= torch.where(torch.rand(4, 256, generator=g) < 0.25, -1.0, 1.0)     # ... some negative (pool at the min row)
    tab[:, 0, 250:] = 0                                    # a = 0
    tab[:, 1] = ri_(-2, 3, (4, 256)) / 2                   # b dyadic; where b = 0 an integer z = 0 is a pre-activation of exactly 0
    tab[:, 1, ::3] = 0
    tab[:, 2] = ri_(-2, 3, (4, 256))                       # mean
    tab[:, 3] = 2.0 ** ri_(-1, 1, (4, 256))                # rstd
    tab[:, 4] = ri_(-1, 2, (4, 256)) / 2                   # m1
    tab[:, 5] = ri_(-1, 2, (4, 256)) / 4                   # m2
    shift4 = ri_(-4, 5, (crops, 256)) / 2
    sel = torch.randint(0, P, (2, crops, 256), generator=g, dtype=torch.int32)
    dsel = ri_(-2, 3, (2, crops, 256)) / 2
    to = lambda t: t.to(dev)                                                             # noqa: E731
    return to(x), [to(w) for w in W], to(tab), to(shift4), to(sel), to(dsel)


def assert_exact_premises(inter, W, tab, shift4, dsel, tf32_passes):
    """every value the kernel forms round-trips through float32, every GEMM operand of the passes in tf32_passes through TF32, and
    every GEMM's sum of magnitudes stays below 2^24 of its product grid, so that every partial sum is exact in any order"""
    vals = dict(inter, W1=W[0], W2=W[1], W3=W[2], W4p=W[3], tab=tab, shift4=shift4, dsel=dsel)
    for k, v in vals.items():
        assert torch.equal(v.double().float().double(), v.double()), k
    # (pass, [(a, b, how)]): how 'w' is a @ w^T (forward), 'd' a @ w (dy = dz W), 't' a^T b (weight gradient); the pairs of one
    # accumulation share their sums
    gemms = [(1, [('x', 'W1', 'w')]), (2, [('y1', 'W2', 'w')]), (3, [('y2', 'W3', 'w')]), (4, [('y2', 'W4p', 'w')]),
             (5, [('dz4', 'y2', 't')]), (5, [('dz3', 'y2', 't')]), (5, [('dz4', 'W4p', 'd'), ('dz3', 'W3', 'd')]),
             (6, [('dz2', 'y1', 't')]), (6, [('dz2', 'W2', 'd')]), (7, [('dz1', 'x', 't')])]
    for p, pairs in gemms:
        S, g = 0, float('inf')
        for a, b, how in pairs:
            if p in tf32_passes:
                for k in (a, b):
                    assert torch.equal(tf32_round(vals[k]), vals[k].double()), (p, k)
            av, bv = vals[a].double().abs(), vals[b].double().abs()
            S = S + {'w': lambda: av @ bv.t(), 'd': lambda: av @ bv, 't': lambda: av.t() @ bv}[how]()
            g = min(g, grid(vals[a]) * grid(vals[b]))
        assert S.max().item() < 2 ** 24 * g, (p, pairs)


# the passes whose GEMM operands are exact in TF32 too: all of them, as the premises check
TF32_EXACT = (1, 2, 3, 4, 5, 6, 7)


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_point_passes_exact_arithmetic(mode):
    """integer points, sparse +-1 weights, power-of-two a and rstd, dyadic b, mean, m1, m2, shift and dsel: every product and partial
    sum is exact in fp32 and every GEMM operand in TF32, so every output equals float64 bit for bit.  Pre-activations of exactly 0
    (b = 0 and an integer z of 0; a = 0) pass no gradient, negative a pools at the min row, and integer z tie often: the extreme rows
    must be the lowest of each tie set.  Two tiles per crop, three crops"""
    crops, P, c0 = 3, 128, 16
    dev = 'cuda'
    x, W, tab, shift4, sel, dsel = exact_inputs(crops, P, c0, dev)
    ref, masks, inter = _pass_ref(x, W, tab, shift4, sel, dsel, P, 'fp32')
    assert_exact_premises(inter, W, tab, shift4, dsel, TF32_EXACT)
    assert any((pre == 0).any() for pre, _ in masks)              # exact zeros at the ReLU threshold
    assert (tab[:, 0] < 0).any() and (tab[:, 0] == 0).any()
    got = run_passes(mode, x, P, W, tab, shift4, sel, dsel)
    for k, (v, _, _, _) in ref.items():
        if k not in ('z3', 'z4'):
            assert torch.equal(got[k].double(), v), (k, (got[k].double() - v).abs().max().item())
    for p in (3, 4):
        z = ref['z%d' % p][0]
        for h, (v, lo) in enumerate(lowest_extreme_rows(z)):
            assert torch.equal(got['x%d' % p][h].double(), v), (p, h)
            assert torch.equal(got['i%d' % p][h].long(), lo), (p, h)
        assert ((z == z.max(1, keepdim=True)[0]).sum(1) > 1).any()   # exact ties between distinct rows


# ---- ties the way production makes them ----------------------------------------------------------------------------------
def tie_points(c0, gen, dev):
    """crops of P = 256 rows: all one row (a box with no point: every sample is the same encoded zero point); n distinct rows then
    one repeated row, for n = 0, 5, 63, 64, 200 (the repeated block starts inside, at the start of and across tiles); one large row
    repeated at rows 10 and 200, the crop's max in some channels and its min in others"""
    P = 256
    crops = []
    crops.append(torch.randn(1, c0, generator=gen, device=dev).expand(P, c0))
    for n in (0, 5, 63, 64, 200):
        c = torch.randn(P, c0, generator=gen, device=dev)
        c[n:] = 3 * torch.randn(1, c0, generator=gen, device=dev)      # large: the extreme row in many channels
        crops.append(c)
    c = torch.randn(P, c0, generator=gen, device=dev)
    c[10] = c[200] = 4 * torch.randn(c0, generator=gen, device=dev)
    crops.append(c)
    return torch.cat(crops).contiguous(), len(crops), P


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_point_passes_at_production_ties(mode):
    """identical rows give identical z in both modes (TF32 included), so the pooled row is the lowest of the repeated rows wherever
    they hold the extreme, across tile boundaries; every output still within its bound"""
    dev = 'cuda'
    gen = torch.Generator(device=dev).manual_seed(31)
    c0 = 32
    W = [torch.randn(n, k, generator=gen, device=dev) / k ** 0.5 for n, k in ((128, c0), (128, 128), (256, 128), (256, 128))]
    tab = random_tab(gen, dev)
    x, crops, P = tie_points(c0, gen, dev)
    shift4 = torch.randn(crops, 256, generator=gen, device=dev)
    sel = torch.randint(0, P, (2, crops, 256), generator=gen, device=dev, dtype=torch.int32)
    dsel = torch.randn(2, crops, 256, generator=gen, device=dev)
    ref, _, _ = _pass_ref(x, W, tab, shift4, sel, dsel, P, mode)
    got = run_passes(mode, x, P, W, tab, shift4, sel, dsel)
    # forward outputs and extremes within their bounds (the backward outputs: the random test, whose masks are kept clear)
    check_against_bounds(mode, got, {k: v for k, v in ref.items() if k in FORWARD})
    starts = [0, 5, 63, 64, 200]
    for p in (3, 4):
        z = ref['z%d' % p][0]
        assert (got['i%d' % p][:, 0] == 0).all() and torch.equal(got['x%d' % p][0, 0], got['x%d' % p][1, 0]), (p, 'padded crop')
        for h in range(2):
            idx = got['i%d' % p][h].long()
            # wherever the device pools in a block of identical rows it pools at the block's first row: the identical rows gave
            # identical z, across tiles.  The block is the extreme in many channels (of the 256)
            for c, n in enumerate(starts, 1):
                inblock = idx[c] >= n
                assert inblock.sum() >= 16 and (idx[c][inblock] == n).all(), (p, h, n, idx[c][inblock].unique().tolist())
            c = len(starts) + 1
            inblock = (idx[c] == 10) | (idx[c] == 200)
            assert inblock.sum() >= 16 and (idx[c][inblock] == 10).all(), (p, h, 'duplicate')


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_tied_rows_give_the_same_gradients(mode):
    """train.py pools a tie at its lowest row: a step on crops of repeated rows gives the same parameter gradients as the float64
    restatement pooled at the lowest, at the highest and at a random row of each tie set (within the step bounds, and the three
    restatements agree among themselves to float64 rounding)"""
    B, L = 2, 8
    seed = SEED + 9
    gen = torch.Generator(device='cuda').manual_seed(seed)
    x, crops, P = tie_points(32, gen, 'cuda')
    pts = torch.cat([x.view(crops, P, 32)] * 3)[:B * L].reshape(B, L, P, 32).contiguous()
    iou = crm_train_ref.crm_train_iou(seed, B, L, box_num=[L, L - 2]).cuda()
    m = crm(mode, seed)
    sd = clone_sd(m)
    _, _, _, grads, _ = step(m, pts, iou)
    rows = {k: v.cpu() for k, v in m.reg.pooled_rows.items()}
    rec = {}
    crm_train_ref.crm_train_step(sd, pts, iou, device='cuda', pooled_rows=rows, record=rec)
    alt = {}
    for how in ('lowest', 'highest', 'random'):
        r = {}
        for k in ('enc1', 'enc2'):
            y = rec[k].cpu()                                         # (crops, P, 256)
            dev_val = y.gather(1, rows[k].long().unsqueeze(1))
            tie = y == dev_val                                       # the tie set of the device's row
            pr = torch.arange(P).view(1, P, 1).expand_as(y)
            if how == 'lowest':
                r[k] = torch.where(tie, pr, P).min(1)[0]
            elif how == 'highest':
                r[k] = torch.where(tie, pr, -1).max(1)[0]
            else:
                key = torch.rand(y.shape, generator=torch.Generator().manual_seed(3)) + tie.double()
                r[k] = key.max(1)[1]
            if how == 'lowest':                                          # the device pools at the lowest row of a positive tie
                pos = dev_val.squeeze(1) > 0
                assert torch.equal(r[k].int()[pos], rows[k][pos]), k
        alt[how] = crm_train_ref.crm_train_step(sd, pts, iou, device='cuda', pooled_rows=r)[1]
    floor = FLOOR * max(g.abs().max().item() for g in alt['lowest'].values())
    for how in ('highest', 'random'):
        for k, g in alt[how].items():
            assert err(g, alt['lowest'][k], floor) <= 1e-10, (how, k)
    _, g32, _ = ref32(sd, pts, iou, mode, pooled_rows=rows)
    ref_err = lambda k, g: err(g, alt['lowest'][k], floor)          # noqa: E731
    check_grads(grads, ref_err, {k: ref_err(k, g) for k, g in g32.items()}, TOL[mode]['grad'])


# ---- what the train-mode point encoders refuse -----------------------------------------------------------------------------
@pytest.mark.parametrize('P,c0,match', [(200, 32, 'multiple of 64'), (100, 32, 'multiple of 64'), (256, 12, 'multiple of 8'),
                                        (256, 72, 'multiple of 8'), (256, 4, 'multiple of 8')])
def test_unsupported_crop_shapes_raise(P, c0, match):
    cfg = ri.crm_cfg()
    m = RefineTemplate(AttrDict({'NAME': 'ConfidenceRefineModel', 'QUERY_POINT_DIMS': c0, 'MEMORY_POINT_DIMS': c0, 'REGRESSION': cfg}))
    m = m.cuda().train()
    pts = torch.randn(1, 4, P, c0, device='cuda')
    with pytest.raises(ValueError, match=match):
        m({'conf_points': pts, 'iou': torch.full((1, 4), 0.9, device='cuda')})


@pytest.mark.parametrize('mlp', [[64, 128], [128, 256], [128, 128, 128]])
def test_unsupported_encoder_mlp_raises(mlp):
    cfg = ri.crm_cfg()
    cfg.ENCODER_MLP = mlp
    m = RefineTemplate(AttrDict({'NAME': 'ConfidenceRefineModel', 'QUERY_POINT_DIMS': 32, 'MEMORY_POINT_DIMS': 32, 'REGRESSION': cfg}))
    m = m.cuda().train()
    with pytest.raises(ValueError, match='ENCODER_MLP'):
        m({'conf_points': torch.randn(1, 4, 64, 32, device='cuda'), 'iou': torch.full((1, 4), 0.9, device='cuda')})

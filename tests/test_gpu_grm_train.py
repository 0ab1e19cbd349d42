"""GRM training on the device (detzero_b200/refine/train.py, csrc/pointmlp_train.cu): one step against the reference's own float64
golden (tests/golden/grm_train.npz) and the float64 restatement (oracle/grm_train_ref.py), each kernel against float64 at every call
train.py makes (random data at derived bounds; exact arithmetic bit for bit), the ties built samples make, a step on samples built
from a tracked sequence, the C ABI's rejections, determinism, dropout, the fp32 / allow_tf32 refusal, the shape check,
train-then-eval and peak memory against autograd."""
import os

import numpy as np
import pytest
import torch

from detzero_b200 import _lib, ops, synthetic
from detzero_b200.config import AttrDict
from detzero_b200.refine import data as rdata, train
from detzero_b200.refine.modules import RefineTemplate
from oracle import grm_train_ref, weights
from oracle import refine_inputs as ri

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'grm_train.npz')
SEED = 7411
U32 = 2.0 ** -24            # fp32 unit roundoff
U_TF32 = 2.0 ** -11         # an operand rounded to nearest TF32 (10 explicit mantissa bits)
TM = ops.PM_TILE            # rows per tile of the train-mode point layers
# Step tolerances.  fp32: the issue's 1e-5 relative on losses and 1e-4 norm-relative (max |error| / max |reference|) on gradients.
# tf32: every point-layer GEMM rounds both operands to TF32, a relative error up to 2 * 2^-11 per product.  Independent roundings
# over a reduction of length K grow like sqrt(K) and are damped by the same 1/sqrt(K) of a BatchNorm-normalised output, so each
# layer adds about 2 * 2^-11 = 1e-3 relative; the memory path chains 5 layers and its BatchNorm statistics, the backward chains the
# same again: 10 * 1e-3 = 1e-2 on gradients, the forward's 5 * 1e-3 = 5e-3 on the losses and running statistics.
TOL = {'fp32': {'loss': 1e-5, 'grad': 1e-4, 'stats': 1e-4},
       'tf32': {'loss': 5e-3, 'grad': 1e-2, 'stats': 5e-3}}
# A bound looser than these, with its cause: the memory path's gradients are sums over B*4096 rows whose terms cancel.  The softmax
# backward makes the key gradient of each query sum to 0 over the 4096 memory rows, and every BatchNorm backward makes dZ sum to 0
# over the rows, so dY5, dZ5 .. dZ1 and their row sums are small remainders of large terms, and a sum of rounded terms keeps the
# rounding of the large ones.  Plain float32 autograd of the same forward (the restatement, run in float32 at the same pooled rows,
# TF32 matmuls in the tf32 mode) has the same conditioning; a gradient is allowed ASSOC times the error that autograd makes on it,
# when that is larger than the bound above.  (Measured at B = 8 in fp32: memory-path gradients 1e-4 to 5e-3, query-path and
# decoder gradients 4e-6.)  ASSOC is measured, not derived: the largest ratio seen was 4.2, on the first position-embedding conv
# weight in tf32 (its gradient sums 24 rows through a BatchNorm backward); 8 leaves room for a different batch.
ASSOC = 8
# BatchNorm biases whose output reaches the loss only through another conv + BatchNorm sum a gradient whose rows add up to 0: their
# gradient is 0 up to rounding, so every gradient's scale is floored at FLOOR times the largest gradient.
FLOOR = 1e-2


def cfg(mode, dropout=0.0):
    c = ri.grm_cfg()
    c.COMPUTE_MODE = mode
    c.DECODER['dropout'] = dropout
    return c


def grm(mode, seed=SEED, dropout=0.0):
    m = RefineTemplate(AttrDict({'NAME': 'GeometryRefineModel', 'QUERY_POINT_DIMS': 11, 'MEMORY_POINT_DIMS': 4,
                                 'REGRESSION': cfg(mode, dropout)}))
    weights.load_seeded(m.reg, seed)
    return m.cuda().train()


def inputs(seed, B, **kw):
    return {k: v.cuda() for k, v in grm_train_ref.grm_train_inputs(seed, B, **kw).items()}


def step(m, inp):
    m.zero_grad(set_to_none=True)
    ret, tb, disp = m(dict(inp))
    ret['loss'].backward()
    grads = {k: p.grad.detach().clone() for k, p in m.reg.named_parameters()}
    stats = {k[4:]: v.detach().clone() for k, v in m.state_dict().items()
             if k.endswith(('running_mean', 'running_var', 'num_batches_tracked'))}
    return ret, tb, disp, grads, stats


def err(got, ref, floor=0.0):
    got, ref = got.double().cpu(), ref.double().cpu()
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), floor)


def autograd_errors(sd, inp, mode, ref, rows, floor):
    """the error of plain float32 (tf32: TF32 matmul) autograd of the restatement on each gradient, against ref"""
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = mode == 'tf32'
    try:
        _, g32, _ = grm_train_ref.grm_train_step(sd, inp, device='cuda', pooled_rows=rows, dtype=torch.float32)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    return {k: ref(k, g) for k, g in g32.items()}


def autograd_record(sd, inp, mode, rows):
    """the record of plain float32 (tf32: TF32 matmul) autograd of the restatement pooled at rows"""
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = mode == 'tf32'
    rec = {}
    try:
        grm_train_ref.grm_train_step(sd, inp, device='cuda', pooled_rows=rows, dtype=torch.float32, record=rec)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    return rec


def path_err(got, ref):
    """the largest error of a point path's output, each channel against its largest value over the rows"""
    scale = ref.abs().amax(dim=0, keepdim=True).clamp_min(1e-30)
    return ((got.to(ref.device).double() - ref).abs() / scale).max().item()


def clone_sd(m):
    return {k[4:]: v.detach().clone() for k, v in m.state_dict().items() if k.startswith('reg.')}


def check_stats(stats, ref, tol):
    for k, v in stats.items():
        if k.endswith('num_batches_tracked'):
            assert int(v) == int(ref[k]) == 1, k
        else:
            assert err(v, ref[k]) <= tol, (k, err(v, ref[k]))


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_matches_reference_golden(mode):
    gold = np.load(GOLD)
    tol = TOL[mode]
    m = grm(mode)
    sd = clone_sd(m)
    inp = inputs(SEED, 2)
    ret, tb, disp, grads, stats = step(m, inp)
    assert set(ret) == {'loss'} and disp == {}
    assert set(tb) == {'cls_loss', 'reg_loss', 'geometry_loss', 'full_loss'}
    for k in ('cls_loss', 'reg_loss', 'geometry_loss'):
        assert abs(tb[k].item() - gold['loss.' + k]) <= tol['loss'] * abs(gold['loss.' + k]), (k, tb[k].item(), gold['loss.' + k])
    assert tb['full_loss'].item() == tb['geometry_loss'].item()
    floor = FLOOR * max(np.abs(gold[k]).max() for k in gold.files if k.startswith('grad.'))

    def gerr(k, g):
        if 'grad.' + k in gold:
            return err(g, torch.from_numpy(gold['grad.' + k]), floor)
        gsq = gold['gsq.' + k]
        p = grm_train_ref.probe(k, g.shape, SEED)
        scale = max(np.sqrt(gsq), floor * np.sqrt(g.numel()))
        return max(abs((g.double() ** 2).sum().item() - gsq) / scale ** 2 / 2,
                   abs((g.double().cpu() * p).sum().item() - gold['gdot.' + k]) / (scale * p.norm().item()))

    errs = {k: gerr(k, g) for k, g in grads.items()}
    ag = autograd_errors(sd, inp, mode, gerr, None, floor)           # float32 autograd pools at its own argmax, as the golden does
    bad = {k: (e, ag[k]) for k, e in errs.items() if e > max(tol['grad'], ASSOC * ag[k])}
    assert not bad, bad
    check_stats(stats, {k[3:]: torch.from_numpy(gold[k]) for k in gold.files if k.startswith('bn.')}, tol['stats'])


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_matches_restatement_at_device_pooled_rows(mode):
    """B = 8 against the float64 restatement pooled at the rows the device picked: arithmetic, without argmax flips"""
    B, seed = 8, SEED + 1
    tol = TOL[mode]
    m = grm(mode, seed)
    sd = clone_sd(m)
    inp = inputs(seed, B)
    inp['geo_query_num'] = torch.tensor([3, 1, 2, 3, 2, 1, 3, 2])
    _, tb, _, grads, stats = step(m, inp)
    rows = {k: v.cpu() for k, v in m.reg.pooled_rows.items()}
    losses, rgrads, rstats = grm_train_ref.grm_train_step(sd, inp, device='cuda', pooled_rows=rows)
    for k, v in losses.items():
        assert abs(tb[k].item() - v) <= tol['loss'] * abs(v), (k, tb[k].item(), v)
    floor = FLOOR * max(g.abs().max().item() for g in rgrads.values())
    errs = {k: err(g, rgrads[k], floor) for k, g in grads.items()}
    ag = autograd_errors(sd, inp, mode, lambda k, g: err(g, rgrads[k], floor), rows, floor)
    bad = {k: (e, ag[k]) for k, e in errs.items() if e > max(tol['grad'], ASSOC * ag[k])}
    assert not bad, bad
    check_stats(stats, rstats, tol['stats'])


def check_pooled_rows(m, sd, inp, mode):
    """every row the device pooled at in the last step of m holds, in float64, a value within the forward bound of the float64
    maximum of its group, and the device pools at a row whose float64 value is below the maximum (a flip: ties, ReLU zeros and
    padded queries included, are not flips) no more often than plain float32 (tf32: TF32) autograd does"""
    rec64, rec32 = {}, {}
    grm_train_ref.grm_train_step(sd, inp, device='cuda', record=rec64)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = mode == 'tf32'
    try:
        grm_train_ref.grm_train_step(sd, inp, device='cuda', dtype=torch.float32, record=rec32)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    for k in ('memory', 'query'):
        y = rec64[k]                                                  # (groups, rows, C) float64 inputs of the max
        dev = m.reg.pooled_rows[k].long()
        top = y.max(dim=1)[0]
        at = y.gather(1, dev.unsqueeze(1)).squeeze(1)
        # the forward's relative error bound (the one the running statistics are held to), on the chosen row and on the maximum
        bound = 2 * TOL[mode]['stats'] * y.abs().amax(dim=1)
        assert ((top - at) <= bound).all(), (k, ((top - at) / bound.clamp_min(1e-30)).max().item())
        at32 = y.gather(1, rec32[k].max(dim=1)[1].unsqueeze(1)).squeeze(1)
        flips_dev, flips_ag = int((at < top).sum()), int((at32 < top).sum())
        assert flips_dev <= 2 * flips_ag + 2, (k, flips_dev, flips_ag, top.numel())


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_pooled_rows_against_float64(mode):
    """B = 8: every row the device pools at holds, in float64, a value within the rounding bound of the float64 maximum of its group,
    and the device picks a row below the float64 maximum no more often than plain float32 (tf32: TF32) autograd does"""
    B, seed = 8, SEED + 1
    m = grm(mode, seed)
    sd = clone_sd(m)
    inp = inputs(seed, B)
    step(m, inp)
    check_pooled_rows(m, sd, inp, mode)


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_is_deterministic(mode):
    inp = inputs(SEED + 2, 4)
    a, b = step(grm(mode), inp), step(grm(mode), inp)
    for k in a[1]:
        assert torch.equal(a[1][k], b[1][k]), k
    for i in (3, 4):
        for k in a[i]:
            assert torch.equal(a[i][k], b[i][k]), k


def test_dropout_changes_the_step_and_stays_finite():
    inp = inputs(SEED + 3, 4)
    torch.manual_seed(0)
    _, tb0, _, g0, _ = step(grm('fp32'), inp)
    torch.manual_seed(0)
    _, tb1, _, g1, _ = step(grm('fp32', dropout=0.1), inp)
    assert torch.isfinite(tb1['geometry_loss']) and all(torch.isfinite(g).all() for g in g1.values())
    assert tb1['geometry_loss'].item() != tb0['geometry_loss'].item()
    assert any(not torch.equal(g0[k], g1[k]) for k in g0)


def test_fp32_refuses_allow_tf32():
    m = grm('fp32')
    inp = inputs(SEED, 2)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        with pytest.raises(RuntimeError, match='allow_tf32'):
            m(dict(inp))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


@pytest.mark.parametrize('mem,qpts', [(4000, 256), (4096, 200)])
def test_unsupported_point_counts_raise(mem, qpts):
    m = grm('tf32')
    with pytest.raises(ValueError, match='multiple of 64'):
        m(dict(inputs(SEED, 2, mem=mem, qpts=qpts)))


@pytest.mark.parametrize('stack,widths', [('QUERY_ENCODER', [96, 128]), ('MEMORY_ENCODER', [128, 192])])
def test_unsupported_channel_widths_raise(stack, widths):
    c = cfg('tf32')
    c[stack] = widths
    m = RefineTemplate(AttrDict({'NAME': 'GeometryRefineModel', 'QUERY_POINT_DIMS': 11, 'MEMORY_POINT_DIMS': 4, 'REGRESSION': c})).cuda().train()
    with pytest.raises(ValueError, match='multiples of 128'):
        m(dict(inputs(SEED, 2)))


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_training_then_eval(mode):
    inp = inputs(SEED + 4, 4)
    m = grm(mode)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    losses = []
    for _ in range(6):
        opt.zero_grad(set_to_none=True)
        ret, _, _ = m(dict(inp))
        ret['loss'].backward()
        opt.step()
        m.update_global_step()
        losses.append(ret['loss'].item())
    assert losses[-1] < losses[0], losses
    m.eval()
    got = m(dict(inp))[0]['pred_boxes']
    fresh = grm(mode).eval()
    fresh.load_state_dict(m.state_dict())
    assert torch.equal(fresh.reg.memory_encoder[1].running_var, m.reg.memory_encoder[1].running_var)
    assert int(fresh.reg.memory_encoder[1].num_batches_tracked) == 6
    ref = fresh(dict(inp))[0]['pred_boxes']
    assert torch.equal(got, ref)


def test_peak_memory_below_autograd():
    B = 128
    inp = inputs(SEED, B)
    m = grm('tf32')
    sd = clone_sd(m)

    def peak(fn):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    step(m, inp)
    m.zero_grad(set_to_none=True)
    dev = peak(lambda: step(m, inp))
    m.zero_grad(set_to_none=True)
    ag = peak(lambda: grm_train_ref.grm_train_step(sd, inp, device='cuda', dtype=torch.float32))
    assert dev < ag, (dev / 2 ** 30, ag / 2 ** 30)


# ---- each kernel against float64 ------------------------------------------------------------------------------------------
# Element bound of a GEMM output: |z - z64| <= (c + (K + 2) u) S, with S = |A| |B| summed over the reduction (the sum of the terms'
# magnitudes), u = 2^-24 for the fp32 accumulation over K terms and the operand's own fp32 arithmetic, c = 0 in fp32 and 2 * 2^-11
# in tf32 (both operands rounded to nearest TF32).
def gamma(mode, K):
    return (0.0 if mode == 'fp32' else 2 * U_TF32) + (K + 2) * U32


# The bound above is the worst case: every term's rounding of the same sign.  Roundings to nearest are nearly independent, so the
# error's root mean square over all elements is held as well to the sum in quadrature, S2 = sum (a b)^2 over the reduction:
# RMS error <= (2 * 2^-11 in tf32 + 2 sqrt(K) 2^-24) sqrt(mean S2).  The RMS of one product's relative error from two operands rounded
# to nearest TF32 is about 0.6 * 2^-11, a third of the operand term; operands rounded two bits coarser would exceed it.
def rms_ok(diff, S2, mode, K):
    c = (0.0 if mode == 'fp32' else 2 * U_TF32) + 2 * K ** 0.5 * U32
    return diff.double().pow(2).mean().sqrt().item() <= c * S2.mean().sqrt().item()


def table(C, gen, dev, neg=True):
    t = torch.zeros(6, C, device=dev)
    t[0] = torch.rand(C, generator=gen, device=dev) + 0.5
    if neg:
        t[0, : C // 4] *= -1                            # negative BN scales: the pooled row is the min row
    t[1] = torch.randn(C, generator=gen, device=dev) * 0.3
    t[2] = torch.randn(C, generator=gen, device=dev) * 0.1
    t[3] = torch.rand(C, generator=gen, device=dev) + 0.5
    t[4:] = torch.randn(2, C, generator=gen, device=dev) * 1e-2
    return t


def act64(x, t):
    t = t.double()
    return (t[0] * x.double() + t[1]).clamp_min(0)


def dz64(dh, z, t):
    t = t.double()
    return t[0] * (dh.double() - t[4] - (z.double() - t[2]) * t[3] * t[5])


# 150 row tiles on 132 SMs: a partial last wave; 3 groups of 3200 rows
R, GS = 150 * 64, 3200
# the production group sizes: a query's 256 points (4 tiles per group) over 152 tiles, a track's 4096 memory points (64 tiles)
ROWS = {GS: R, 256: 152 * 64, 4096: 3 * 4096}


# (K, N, with_act, shift, gsize): the two cases at 3200-row groups, then every forward call of train.py: the query path's
# 4 -> 128 (exact fp32 in both modes in train.py, both modes here), 128 -> 128 and the pooled 128 -> 256; the memory path's
# 11 -> 128, 128 -> 128, the pooled 128 -> 512, the 128 + per-track shift -> 512 and 512 -> 256
@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
@pytest.mark.parametrize('K,N,with_act,shifted,gsize', [
    pytest.param(11, 512, False, False, GS, id='11-False'), pytest.param(128, 512, True, True, GS, id='128-True'),
    (4, 128, False, False, 256), (128, 128, True, False, 256), (128, 256, True, False, 256),
    (11, 128, False, False, 4096), (128, 128, True, False, 4096), (128, 512, True, False, 4096), (128, 512, True, True, 4096),
    (512, 256, True, False, 4096)])
def test_forward_kernel_against_float64(mode, K, N, with_act, shifted, gsize):
    dev = 'cuda'
    gen = torch.Generator(device=dev).manual_seed(11)
    R, GS = ROWS[gsize], gsize
    G = R // GS
    x = torch.randn(R, K, generator=gen, device=dev)
    # exact ties: rows repeated within each group, one of them made the group's largest row
    for g in range(G):
        x[g * GS + GS * 5 // 8] = x[g * GS + 100] = 3 * x[g * GS + 100].abs()
        x[g * GS + GS - 100] = x[g * GS + 7]
    tin = table(K, gen, dev, neg=False) if with_act else None
    w = torch.randn(N, K, generator=gen, device=dev) / K ** 0.5
    shift = torch.randn(G, N, generator=gen, device=dev) if shifted else None
    z, ps, ev, ei = ops.pm_fwd(x, w, _lib.MODES[mode], tin, shift=shift, gsize=GS, ext=True)
    a = act64(x, tin) if with_act else x.double()
    ref = a @ w.double().t()
    S = a.abs() @ w.double().abs().t()
    if shift is not None:
        ref = ref + shift.double().repeat_interleave(GS, 0)
        S = S + shift.double().abs().repeat_interleave(GS, 0)
    assert ((z.double() - ref).abs() <= gamma(mode, K) * S).all()
    S2 = a.pow(2) @ w.double().pow(2).t()
    assert rms_ok(z.double() - ref, S2, mode, K)
    # the statistics are float64 sums of the z written
    tot = ops.pm_reduce_tiles(ps)[0]
    zd = z.double()
    assert torch.allclose(tot[0], zd.sum(0), rtol=1e-12, atol=1e-9 * zd.abs().sum(0).max().item())
    assert torch.allclose(tot[1], (zd * zd).sum(0), rtol=1e-12, atol=0)
    # extremes: exactly the max / min of the z written, at its lowest row
    zext, iext = ops.pm_group_ext(ev, ei, G)
    zc = z.view(G, GS, N).cpu().numpy()
    assert np.array_equal(zext[0].cpu().numpy(), zc.max(1)) and np.array_equal(zext[1].cpu().numpy(), zc.min(1))
    assert np.array_equal(iext[0].cpu().numpy(), zc.argmax(1)) and np.array_equal(iext[1].cpu().numpy(), zc.argmin(1))
    # the pooled row's float64 value lies within the rounding bound of the float64 extreme of its group (twice the element bound:
    # both the chosen row and the true extreme carry one)
    r64, s64 = ref.view(G, GS, N), S.view(G, GS, N)
    for h, (fn, idx) in enumerate(((torch.max, iext[0]), (torch.min, iext[1]))):
        at = r64.gather(1, idx.long().unsqueeze(1)).squeeze(1)
        bound = 2 * gamma(mode, K) * s64.max(1)[0]
        assert ((at - fn(r64, 1)[0]).abs() <= bound).all(), h


# (segments [(N, pooled)], Kout, gsize): the memory path's y2 gradient at 3200-row groups (the two parameter sets named by mode
# alone), then every dgrad call of train.py: dh4 (dense 256 -> 512), dh2 of the memory path (pooled 512 + dense 512 -> 128 at 4096),
# dh1 (dense 128 -> 128), dh2 of the query path (pooled 256 -> 128 at 256); and one pooled segment into 512 at 4096
DGRAD = [((((512, True), (512, False)), 128, GS), ''), ((((256, False),), 512, 4096), 'dh4'),
         ((((512, True), (512, False)), 128, 4096), 'mem-dh2'), ((((128, False),), 128, 4096), 'dh1'),
         ((((256, True),), 128, 256), 'query-dh2'), ((((512, True),), 512, 4096), 'pooled-512')]


@pytest.mark.parametrize('mode,case', [pytest.param(m, c, id='-'.join(filter(None, (i, m)))) for c, i in DGRAD for m in ('fp32', 'tf32')])
def test_dgrad_kernel_against_float64(mode, case):
    """dH of the layer below from one or two layers' dZ, dense or pooled, with the layer below's sums"""
    dev = 'cuda'
    gen = torch.Generator(device=dev).manual_seed(12)
    segs, Kout, GS = case
    R = ROWS[GS]
    G = R // GS
    arg, d, Ws = [], [], []
    for N, pooled in segs:
        z = torch.randn(R, N, generator=gen, device=dev)
        t = table(N, gen, dev)
        if pooled:
            sel = torch.randint(0, GS, (G, N), generator=gen, device=dev, dtype=torch.int32)
            dsel = torch.randn(G, N, generator=gen, device=dev)
            dh = pooled_dh(sel, dsel, GS)
        else:
            sel = dsel = None
            dh = torch.randn(R, N, generator=gen, device=dev)
        W = torch.randn(N, Kout, generator=gen, device=dev) / N ** 0.5
        arg.append((None if pooled else dh, sel, dsel, z, t, W.t().contiguous()))
        d.append(dz64(dh, z, t))
        Ws.append(W.double())
    zl = torch.randn(R, Kout, generator=gen, device=dev)
    tl = table(Kout, gen, dev)
    dh, ps = ops.pm_dgrad(arg, zl, tl, _lib.MODES[mode], gsize=GS)
    dy = sum(a @ W for a, W in zip(d, Ws))
    S = sum(a.abs() @ W.abs() for a, W in zip(d, Ws))
    Ktot = sum(N for N, _ in segs)
    pre = tl[0].double() * zl.double() + tl[1].double()
    keep = pre.abs() > 1e-5                             # a mask taken within fp32 rounding of 0 may go either way
    ref = dy * (pre > 0)
    assert ((dh.double() - ref).abs() <= gamma(mode, Ktot + 8) * S)[keep].all()
    S2 = sum(a.pow(2) @ W.pow(2) for a, W in zip(d, Ws)) * (pre > 0)
    assert rms_ok((dh.double() - ref)[keep], S2[keep], mode, Ktot)
    tot = ops.pm_reduce_tiles(ps)[0]
    xh = (zl.double() - tl[2].double()) * tl[3].double()
    hd = dh.double()
    assert torch.allclose(tot[0], hd.sum(0), rtol=1e-12, atol=1e-12 * hd.abs().sum(0).max().item())
    assert ((tot[1] - (hd * xh).sum(0)).abs() <= 4 * U32 * (hd * xh).abs().sum(0)).all()


# (N, K, pooled, with_act, gsize): three cases at 3200-row groups, then every weight gradient of train.py: the query path's dW1
# (K = 4), dW2 and pooled dW3 at 256; the memory path's dW1 (K = 11), dW2, pooled dW3, dW4p and dW5 (K = 512) at 4096
@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
@pytest.mark.parametrize('N,K,pooled,with_act,gsize', [
    pytest.param(512, 128, True, True, GS, id='512-128-True-True'), pytest.param(256, 512, False, True, GS, id='256-512-False-True'),
    pytest.param(128, 11, False, False, GS, id='128-11-False-False'),
    (128, 4, False, False, 256), (128, 128, False, True, 256), (256, 128, True, True, 256),
    (128, 11, False, False, 4096), (128, 128, False, True, 4096), (512, 128, True, True, 4096), (512, 128, False, True, 4096),
    (256, 512, False, True, 4096)])
def test_wgrad_kernel_against_float64(mode, N, K, pooled, with_act, gsize):
    dev = 'cuda'
    gen = torch.Generator(device=dev).manual_seed(13)
    R, GS = ROWS[gsize], gsize
    G = R // GS
    z = torch.randn(R, N, generator=gen, device=dev)
    t = table(N, gen, dev)
    x = torch.randn(R, K, generator=gen, device=dev)
    tin = table(K, gen, dev) if with_act else None
    if pooled:
        sel = torch.randint(0, GS, (G, N), generator=gen, device=dev, dtype=torch.int32)
        dsel = torch.randn(G, N, generator=gen, device=dev)
        dh = torch.zeros(R, N, device=dev, dtype=torch.float64)
        dh.scatter_(0, sel.long() + GS * torch.arange(G, device=dev).unsqueeze(1), dsel.double())
        seg = (None, sel, dsel, z, t)
    else:
        dh = torch.randn(R, N, generator=gen, device=dev)
        seg = (dh, None, None, z, t)
    dw = ops.pm_wgrad(seg, x, _lib.MODES[mode], tin, gsize=GS)
    d = dz64(dh, z, t)
    a = act64(x, tin) if with_act else x.double()
    ref = d.t() @ a
    S = d.abs().t() @ a.abs()
    # fp32 partial sums over at most R rows per CTA, then a float64 sum
    assert ((dw - ref).abs() <= gamma(mode, R + 8) * S).all()
    assert rms_ok(dw - ref, d.pow(2).t() @ a.pow(2), mode, R)


# ---- exact arithmetic: every value the kernels form is representable, so fp32 and TF32 must both give float64's bits ---------------
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


def tile_sums64(u, v):
    """per 64-row tile column sums of u and v: (R / 64, 2, N)"""
    R, N = u.shape
    return torch.stack([u.view(R // TM, TM, N).sum(1), v.view(R // TM, TM, N).sum(1)], 1)


def lowest_extremes(z, gsize):
    """per group of gsize rows and column of z (R, N): [max, min] (2, groups, N) and the lowest row in the group holding each"""
    zg = z.view(-1, gsize, z.shape[1])
    r = torch.arange(gsize, device=z.device).view(1, gsize, 1)
    vals, rows = [], []
    for v in (zg.max(1)[0], zg.min(1)[0]):
        vals.append(v)
        rows.append(torch.where(zg == v.unsqueeze(1), r, gsize).min(1)[0])
    return torch.stack(vals), torch.stack(rows)


def pooled_dh(sel, dsel, gsize):
    """the dense (R, N) float64 dH of a pooled gradient: dsel at row sel of each group, 0 elsewhere"""
    G, N = sel.shape
    dh = torch.zeros(G * gsize, N, dtype=torch.float64, device=sel.device)
    dh.scatter_(0, sel.long() + gsize * torch.arange(G, device=sel.device).unsqueeze(1), dsel.double())
    return dh


class Chain:
    """the float64 statement of one GRM point path, layer by layer as train.py calls the kernels, and the same calls on the device.
    Each device call is fed the float64 values of its inputs (rounded to float32), so every output is compared on its own.
    x (R, c0) the points, W [W1, W2, W3 (+ W4p, W5 for the memory path)] (out, in), tab (layers, 6, 512) per-layer tables, shift
    (groups, 512) the memory path's per-track shift, sel / dsel (groups, C3) the pooled gradient of layer 3, dy (R, 256) the memory
    path's output gradient"""

    def __init__(self, x, W, tab, gsize, shift=None, sel=None, dsel=None, dy=None):
        d = lambda t: None if t is None else t.double()                          # noqa: E731
        self.x, self.W, self.gsize = d(x), [d(w) for w in W], gsize
        self.tab = [d(tab[l, :, :w.shape[0]]) for l, w in enumerate(W)]         # layer l's table over its own channels
        self.shift, self.sel, self.dsel, self.dy = d(shift), sel, d(dsel), d(dy)
        self.mem = len(W) == 5
        self.calls = {}

    @staticmethod
    def act(z, t):
        return (t[0] * z + t[1]).clamp_min(0)

    @staticmethod
    def dz(dh, z, t):
        return t[0] * (dh - t[4] - ((z - t[2]) * t[3]) * t[5])

    @staticmethod
    def dgrad(segs, zl, tl):
        dy = sum(Chain.dz(dh, z, t) @ W for dh, z, t, W in segs)
        dh = dy * (tl[0] * zl + tl[1] > 0)
        return dh, tile_sums64(dh, dh * ((zl - tl[2]) * tl[3]))

    def reference(self):
        """{call: {output: float64 value}} and the values the kernels form on the way, for the premises"""
        x, (W1, W2, W3), t, G = self.x, self.W[:3], self.tab, self.gsize
        out, formed, gemms = {}, {}, []
        z1 = x @ W1.t()
        y1 = self.act(z1, t[0])
        z2 = y1 @ W2.t()
        y2 = self.act(z2, t[1])
        z3 = y2 @ W3.t()
        out['fwd1'] = {'z': z1, 'ps': tile_sums64(z1, z1 * z1)}
        out['fwd2'] = {'z': z2, 'ps': tile_sums64(z2, z2 * z2)}
        ev, ei = lowest_extremes(z3, TM)                                       # per tile, the row within the group
        ei = ei + (torch.arange(ei.shape[1], device=ei.device) * TM % G).view(1, -1, 1)
        out['fwd3'] = {'z': z3, 'ps': tile_sums64(z3, z3 * z3), 'ev': ev.transpose(0, 1), 'ei': ei.transpose(0, 1)}
        out['ext3'] = dict(zip(('zext', 'iext'), lowest_extremes(z3, G)))
        gemms += [('x', 'W1', 'w'), ('y1', 'W2', 'w'), ('y2', 'W3', 'w')]
        formed.update(x=x, z1=z1, pre1=t[0][0] * z1 + t[0][1], y1=y1, z2=z2, pre2=t[1][0] * z2 + t[1][1], y2=y2, z3=z3,
                      W1=W1, W2=W2, W3=W3)
        dh3 = pooled_dh(self.sel, self.dsel, G)
        dz3 = self.dz(dh3, z3, t[2])
        formed.update(dz3=dz3, xh3=(z3 - t[2][2]) * t[2][3], dsel=self.dsel)
        segs = [(dh3, z3, t[2], W3)]
        wg = {'w3': (dz3, y2)}
        if self.mem:
            W4p, W5 = self.W[3:]
            z4 = y2 @ W4p.t() + self.shift.repeat_interleave(G, 0)
            y4 = self.act(z4, t[3])
            z5 = y4 @ W5.t()
            out['fwd4'] = {'z': z4, 'ps': tile_sums64(z4, z4 * z4)}
            out['red4'] = {'out': tile_sums64(z4, z4 * z4).view(-1, G // TM, 2, z4.shape[1]).sum(1)}
            out['fwd5'] = {'z': z5, 'ps': tile_sums64(z5, z5 * z5)}
            out['act5'] = {'y': self.act(z5, t[4])}
            dh5 = self.dy * (t[4][0] * z5 + t[4][1] > 0)
            out['dh5'] = {'dh': dh5, 'ps': tile_sums64(dh5, dh5 * ((z5 - t[4][2]) * t[4][3]))}
            dz5 = self.dz(dh5, z5, t[4])
            dh4, ps4 = self.dgrad([(dh5, z5, t[4], W5)], z4, t[3])
            out['dgrad4'] = {'dh': dh4, 'ps': ps4}
            out['red_dh4'] = {'out': ps4.view(-1, G // TM, 2, z4.shape[1]).sum(1)}
            dz4 = self.dz(dh4, z4, t[3])
            segs.append((dh4, z4, t[3], W4p))
            wg.update(w5=(dz5, y4), w4p=(dz4, y2))
            gemms += [('y2', 'W4p', 'w'), ('y4', 'W5', 'w'), ('dz5', 'W5', 'd'), ('dz5', 'y4', 't'), ('dz4', 'y2', 't')]
            formed.update(z4=z4, pre4=t[3][0] * z4 + t[3][1], y4=y4, z5=z5, pre5=t[4][0] * z5 + t[4][1], y5=out['act5']['y'], W4p=W4p,
                          W5=W5, shift=self.shift, dy=self.dy, dh5=dh5, xh5=(z5 - t[4][2]) * t[4][3], dz5=dz5, dh4=dh4,
                          xh4=(z4 - t[3][2]) * t[3][3], dz4=dz4)
        dh2, ps2 = self.dgrad(segs, z2, t[1])
        out['dgrad2'] = {'dh': dh2, 'ps': ps2}
        dz2 = self.dz(dh2, z2, t[1])
        dh1, ps1 = self.dgrad([(dh2, z2, t[1], W2)], z1, t[0])
        out['dgrad1'] = {'dh': dh1, 'ps': ps1}
        dz1 = self.dz(dh1, z1, t[0])
        wg.update(w2=(dz2, y1), w1=(dz1, x))
        for k, (a, b) in wg.items():
            out[k] = {'dw': a.t() @ b}
        gemms.append([('dz3', 'W3', 'd')] + ([('dz4', 'W4p', 'd')] if self.mem else []))
        gemms += [('dz2', 'W2', 'd'), ('dz3', 'y2', 't'), ('dz2', 'y1', 't'), ('dz1', 'x', 't')]
        formed.update(dh2=dh2, xh2=(z2 - t[1][2]) * t[1][3], dz2=dz2, dh1=dh1, xh1=(z1 - t[0][2]) * t[0][3], dz1=dz1)
        for l, tl in enumerate(t):
            formed['tab%d' % l] = tl
        # the terms of dZ = a (dH - m1 - xhat m2) as the kernels form them
        for l, (dh, z) in {2: (dh3, z3), 1: (dh2, z2), 0: (dh1, z1)}.items():
            tl = t[l]
            formed['dz_terms%d' % l] = torch.cat([z - tl[2], dh - tl[4], ((z - tl[2]) * tl[3]) * tl[5], dh - tl[4] - ((z - tl[2]) * tl[3]) * tl[5]])
        return out, formed, gemms

    def device(self, mode):
        """the same calls on the device: {call: {output: tensor}}"""
        f = lambda t: None if t is None else t.float().contiguous()             # noqa: E731
        md, G, t = _lib.MODES[mode], self.gsize, [f(tl) for tl in self.tab]
        groups = self.x.shape[0] // G
        x, (W1, W2, W3) = f(self.x), [f(w) for w in self.W[:3]]
        ref, _, _ = self.reference()
        z1, z2, z3 = (f(ref['fwd%d' % i]['z']) for i in (1, 2, 3))
        got = {}
        got['fwd1'] = dict(zip(('z', 'ps'), ops.pm_fwd(x, W1, md)[:2]))
        got['fwd2'] = dict(zip(('z', 'ps'), ops.pm_fwd(z1, W2, md, t[0])[:2]))
        z, ps, ev, ei = ops.pm_fwd(z2, W3, md, t[1], gsize=G, ext=True)
        got['fwd3'] = {'z': z, 'ps': ps, 'ev': ev, 'ei': ei}
        got['ext3'] = dict(zip(('zext', 'iext'), ops.pm_group_ext(f(ref['fwd3']['ev']), ref['fwd3']['ei'].int().contiguous(), groups)))
        sel, dsel = self.sel.int().contiguous(), f(self.dsel)
        segs = [(None, sel, dsel, z3, t[2], W3.t().contiguous())]
        wg = {'w3': ((None, sel, dsel, z3, t[2]), z2, t[1])}
        if self.mem:
            W4p, W5 = (f(w) for w in self.W[3:])
            z4, z5 = f(ref['fwd4']['z']), f(ref['fwd5']['z'])
            got['fwd4'] = dict(zip(('z', 'ps'), ops.pm_fwd(z2, W4p, md, t[1], shift=f(self.shift), gsize=G)[:2]))
            got['red4'] = {'out': ops.pm_reduce_tiles(ref['fwd4']['ps'].contiguous(), groups)}
            got['fwd5'] = dict(zip(('z', 'ps'), ops.pm_fwd(z4, W5, md, t[3])[:2]))
            got['act5'] = {'y': ops.pm_act(z5, t[4])}
            got['dh5'] = dict(zip(('dh', 'ps'), ops.pm_dh(f(self.dy), z5, t[4])))
            dh5, dh4 = f(ref['dh5']['dh']), f(ref['dgrad4']['dh'])
            got['dgrad4'] = dict(zip(('dh', 'ps'), ops.pm_dgrad([(dh5, None, None, z5, t[4], W5.t().contiguous())], z4, t[3], md)))
            got['red_dh4'] = {'out': ops.pm_reduce_tiles(ref['dgrad4']['ps'].contiguous(), groups)}
            segs.append((dh4, None, None, z4, t[3], W4p.t().contiguous()))
            wg.update(w5=((dh5, None, None, z5, t[4]), z4, t[3]), w4p=((dh4, None, None, z4, t[3]), z2, t[1]))
        got['dgrad2'] = dict(zip(('dh', 'ps'), ops.pm_dgrad(segs, z2, t[1], md, gsize=G)))
        dh2, dh1 = f(ref['dgrad2']['dh']), f(ref['dgrad1']['dh'])
        got['dgrad1'] = dict(zip(('dh', 'ps'), ops.pm_dgrad([(dh2, None, None, z2, t[1], W2.t().contiguous())], z1, t[0], md)))
        wg.update(w2=((dh2, None, None, z2, t[1]), z1, t[0]), w1=((dh1, None, None, z1, t[0]), x, None))
        for k, (seg, xin, tin) in wg.items():
            got[k] = {'dw': ops.pm_wgrad(seg, xin, md, tin, gsize=G)}
        return got


def exact_chain(mem, dev):
    """integer points in {-1, 0, 1}, sparse +-1 weights, power-of-two a and rstd (a = 0 and negative a on some channels), dyadic b
    (0 on every third channel, so an integer z of 0 is a pre-activation of exactly 0), mean, m1, m2, shift, dsel and dy.  The memory
    path at 640 rows per track (10 tiles: the two-level tile reduction), the query path at 256 rows per query (4 tiles)"""
    g = torch.Generator(device='cpu').manual_seed(79 + mem)
    ri_ = lambda lo, hi, shape: torch.randint(lo, hi, shape, generator=g).float()       # noqa: E731

    def sparse_w(n, k, per):                              # per nonzeros of +-1 in each output row
        w = torch.zeros(n, k)
        for i in range(n):
            w[i, torch.randperm(k, generator=g)[:per]] = ri_(0, 2, (per,)) * 2 - 1
        return w

    if mem:
        G, groups, c0 = 640, 2, 11
        W = [sparse_w(128, c0, 3), sparse_w(128, 128, 1), sparse_w(512, 128, 2), sparse_w(512, 128, 2), sparse_w(256, 512, 2)]
    else:
        G, groups, c0 = 256, 3, 4
        W = [sparse_w(128, c0, 3), sparse_w(128, 128, 2), sparse_w(256, 128, 2)]
    L = len(W)
    x = ri_(-1, 2, (groups * G, c0))
    tab = torch.zeros(L, 6, 512)
    tab[:, 0] = 2.0 ** ri_(-1, 1, (L, 512))                 # a: powers of two ...
    tab[:, 0] *= torch.where(torch.rand(L, 512, generator=g) < 0.25, -1.0, 1.0)      # ... some negative (pool at the min row)
    tab[:, 0, 100:104] = 0                                  # a = 0
    tab[:, 1] = ri_(-2, 3, (L, 512)) / 2                    # b dyadic
    tab[:, 1, ::3] = 0
    tab[:, 2] = ri_(-2, 3, (L, 512))                        # mean
    tab[:, 3] = 2.0 ** ri_(0, 2, (L, 512))                  # rstd
    tab[:, 4] = ri_(-1, 2, (L, 512)) / 2                    # m1
    tab[:, 5] = ri_(-1, 2, (L, 512))                        # m2
    C3 = W[2].shape[0]
    sel = torch.randint(0, G, (groups, C3), generator=g, dtype=torch.int32)
    dsel = ri_(-2, 3, (groups, C3)) / 2
    shift = ri_(-4, 5, (groups, 512)) / 2 if mem else None
    dy = ri_(-1, 2, (groups * G, 256)) / 2 if mem else None
    to = lambda t: None if t is None else t.to(dev)                                      # noqa: E731
    return Chain(to(x), [to(w) for w in W], to(tab), G, to(shift), to(sel), to(dsel), to(dy))


def assert_exact_premises(chain):
    """every value the kernels form round-trips through float32, every GEMM operand through TF32, and every GEMM's sum of magnitudes
    stays below 2^24 of its product grid, so that every partial sum is exact in any order and the float64 sums are exact too"""
    out, formed, gemms = chain.reference()
    for k, v in formed.items():
        assert torch.equal(v.double().float().double(), v.double()), k
    for k, calls in out.items():                              # the float32 outputs (the sums are float64)
        for o, v in calls.items():
            if o in ('z', 'dh', 'y', 'ev', 'zext'):
                assert torch.equal(v.double().float().double(), v.double()), (k, o)
    for pairs in gemms:
        pairs = pairs if isinstance(pairs, list) else [pairs]
        S, gr = 0, float('inf')
        for a, b, how in pairs:
            for k in (a, b):
                assert torch.equal(tf32_round(formed[k]), formed[k].double()), k
            av, bv = formed[a].abs(), formed[b].abs()
            S = S + {'w': lambda: av @ bv.t(), 'd': lambda: av @ bv, 't': lambda: av.t() @ bv}[how]()
            gr = min(gr, grid(formed[a]) * grid(formed[b]))
        assert S.max().item() < 2 ** 24 * gr, (pairs, S.max().item(), gr)
    return out, formed


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
@pytest.mark.parametrize('path', ['memory', 'query'])
def test_kernels_exact_arithmetic(mode, path):
    """every value the kernels form is exact in fp32 and every GEMM operand in TF32 (the test asserts it), so every output of every
    call train.py makes equals float64 bit for bit: z, the tile sums and extremes, the group extremes, the per-track sums, dH and its
    sums, the weight gradients, dh5 and y5.  Pre-activations of exactly 0 pass no gradient, a = 0 and negative a occur, and integer z
    tie often: every extreme row must be the lowest of its tie set"""
    chain = exact_chain(path == 'memory', 'cuda')
    ref, formed = assert_exact_premises(chain)
    assert (formed['pre1'] == 0).any() and (formed['pre2'] == 0).any()            # exact zeros at the ReLU threshold
    assert (formed['tab2'][0] < 0).any() and (formed['tab2'][0] == 0).any()
    got = chain.device(mode)
    assert set(got) == set(ref)
    for call, outs in ref.items():
        for k, v in outs.items():
            g = got[call][k]
            if k in ('ei', 'iext'):                                                 # rows within the group
                assert torch.equal(g.long(), v.long()), (path, call, k, int((g.long() != v.long()).sum()))
            else:
                assert torch.equal(g.double(), v), (path, call, k, (g.double() - v).abs().max().item())
    zext = ref['ext3']['zext']
    z3 = formed['z3'].view(-1, chain.gsize, zext.shape[-1])
    assert ((z3 == zext[0].unsqueeze(1)).sum(1) > 1).any() and ((z3 == zext[1].unsqueeze(1)).sum(1) > 1).any()   # ties


# ---- the elementwise calls and the per-group reductions ---------------------------------------------------------------------
@pytest.mark.parametrize('N', [256, 512])
def test_dh_and_act_kernels_against_float64(N):
    """dh5 = dY [a z + b > 0] is dY or 0 exactly where the mask is clear of rounding, its per-tile sums within a float64 sum's and
    xhat's fp32 rounding; y5 = ReLU(a z + b) within one fp32 rounding of the fma"""
    dev = 'cuda'
    gen = torch.Generator(device=dev).manual_seed(14)
    R = 150 * 64
    z = torch.randn(R, N, generator=gen, device=dev)
    t = table(N, gen, dev)
    t[0, 5] = 0                                         # a = 0: the mask is b > 0
    dy = torch.randn(R, N, generator=gen, device=dev)
    dh, ps = ops.pm_dh(dy, z, t)
    pre = t[0].double() * z.double() + t[1].double()
    keep = pre.abs() > 1e-5
    ref = dy.double() * (pre > 0)
    assert torch.equal(dh.double()[keep], ref[keep])
    assert ((dh == dy) | (dh == 0)).all()
    xh = (z.double() - t[2].double()) * t[3].double()
    hd = dh.double()
    sums = tile_sums64(hd, hd * xh)
    assert ps.shape == sums.shape
    assert ((ps[:, 0] - sums[:, 0]).abs() <= TM * 2.0 ** -53 * tile_sums64(hd.abs(), hd.abs())[:, 0]).all()
    assert ((ps[:, 1] - sums[:, 1]).abs() <= 4 * U32 * tile_sums64(hd.abs(), (hd * xh).abs())[:, 1]).all()
    y = ops.pm_act(z, t)
    ya = act64(z, t)
    assert ((y.double() - ya).abs() <= U32 * pre.abs()).all()
    assert (y >= 0).all() and torch.equal(y[:, 5], torch.full_like(y[:, 5], max(t[1, 5].item(), 0.0)))


@pytest.mark.parametrize('tpg', [64, 150])
def test_reduce_tiles_per_group_against_float64(tpg):
    """the per-track sums train.py takes with groups = B (zsum4 and pg): 64 tiles per group in one pass, and 150, which takes the
    two-level reduction (runs of 2 tiles, then the run sums); each group's sum within a float64 sum's rounding"""
    dev = 'cuda'
    gen = torch.Generator(device=dev).manual_seed(15 + tpg)
    G, N = 5, 512
    ps = torch.randn(G * tpg, 2, N, generator=gen, device=dev, dtype=torch.float64) + 0.5
    ps[:, :, :7] = torch.arange(G * tpg, device=dev, dtype=torch.float64).view(-1, 1, 1)     # exact integer tile ids
    out = ops.pm_reduce_tiles(ps, G)
    ref = ps.view(G, tpg, 2, N).sum(1)
    assert out.shape == (G, 2, N)
    assert ((out - ref).abs() <= tpg * 2.0 ** -52 * ps.abs().view(G, tpg, 2, N).sum(1)).all()
    assert torch.equal(out[:, :, :7], ref[:, :, :7])                    # each group its own tiles, exactly


# ---- ties the way built samples make them ----------------------------------------------------------------------------------
def tie_groups(P, c0, gen, dev, far, zero, span=None):
    """groups of P rows: one repeated row (a padded query when zero: all zero), n distinct rows then one large row repeated over
    span rows (to the end by default), for n = 5, 63, 64 and P * 5 // 8 + 3 (the repeated block starts inside a tile, at a tile
    start and across tile boundaries), one large row repeated at rows 10 and far.  Returns (rows, [(group, block start or None,
    block end)])"""
    groups, blocks = [], []
    if zero:
        groups.append(torch.zeros(P, c0, device=dev))
        blocks.append((len(groups) - 1, 0, P))
    groups.append(torch.randn(1, c0, generator=gen, device=dev).expand(P, c0))
    blocks.append((len(groups) - 1, 0, P))
    for n in (5, 63, 64, P * 5 // 8 + 3):
        c = torch.randn(P, c0, generator=gen, device=dev)
        end = P if span is None else n + span
        c[n:end] = 3 * torch.randn(1, c0, generator=gen, device=dev)
        groups.append(c)
        blocks.append((len(groups) - 1, n, end))
    c = torch.randn(P, c0, generator=gen, device=dev)
    c[10] = c[far] = 4 * torch.randn(c0, generator=gen, device=dev)
    groups.append(c)
    blocks.append((len(groups) - 1, None, None))
    return torch.cat(groups).contiguous(), blocks


def check_block_rows(idx, blocks, P, far, what):
    """idx (2 or 1, groups, C): wherever a group pools in its repeated block it pools at the block's first row"""
    for g, n, end in blocks:
        i = idx[:, g]
        if n == 0:
            assert (i == 0).all(), (what, g, 'repeated row')
        elif n is not None:
            inb = (i >= n) & (i < end)
            assert inb.sum() >= 16 and (i[inb] == n).all(), (what, g, n, i[inb].unique().tolist())
        else:
            inb = (i == 10) | (i == far)
            assert inb.sum() >= 16 and (i[inb] == 10).all(), (what, g, 'far apart')


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
@pytest.mark.parametrize('path', ['memory', 'query'])
def test_group_extremes_at_built_sample_ties(mode, path):
    """the memory path's 4096-row groups and the query path's 256-row groups through layers 1 - 3 and pm_group_ext: identical rows
    give identical z in both modes, so each group's max and min lie at the first row of a repeated block wherever the block holds
    them, across tiles; an all-zero query gives z1 = 0 exactly"""
    dev = 'cuda'
    gen = torch.Generator(device=dev).manual_seed(32)
    P, c0, C3 = (4096, 11, 512) if path == 'memory' else (256, 4, 256)
    far = P - 56
    x, blocks = tie_groups(P, c0, gen, dev, far, zero=path == 'query')
    md = _lib.MODES[mode]
    W = [torch.randn(n, k, generator=gen, device=dev) / k ** 0.5 for n, k in ((128, c0), (128, 128), (C3, 128))]
    t1, t2 = table(128, gen, dev), table(128, gen, dev)
    z1 = ops.pm_fwd(x, W[0], _lib.DZ_F32)[0]
    if path == 'query':
        assert (z1[:P] == 0).all()
    z2 = ops.pm_fwd(z1, W[1], md, t1)[0]
    z3, _, ev, ei = ops.pm_fwd(z2, W[2], md, t2, gsize=P, ext=True)
    zext, iext = ops.pm_group_ext(ev, ei, x.shape[0] // P)
    vals, rows = lowest_extremes(z3, P)
    assert torch.equal(zext.double(), vals.double()) and torch.equal(iext.long(), rows)
    check_block_rows(iext.long(), blocks, P, far, path)


def tie_inputs(seed):
    """a GRM batch whose memory tracks and queries are the tie groups: B = 6 tracks of 4096 memory rows, Q = 3 queries of 256 rows
    with geo_query_num [1, 3, 3, 3, 3, 2], the padded queries all zero as the builders make them"""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    B, Q, P, N = 6, 3, 256, 4096
    inp = inputs(seed, B)
    # memory blocks of 300 rows: blocks to the end of a 4096-row track would leave the batch a handful of distinct rows, whose
    # BatchNorm variances are the small remainders of large terms (a conditioning of the inputs, not of the ties)
    mem, mblocks = tie_groups(N, 11, gen, 'cuda', N - 56, zero=False, span=300)
    q, qblocks = tie_groups(P, 4, gen, 'cuda', P - 56, zero=True)
    qp = inp['geo_query_points'].reshape(B * Q, P, 4).clone()
    num = torch.tensor([1, 3, 3, 3, 3, 2])
    pad = torch.arange(Q)[None] >= num[:, None]
    pad_groups = pad.reshape(-1).nonzero()[:, 0].tolist()                          # 1, 2, 17
    live = [g for g in range(B * Q) if g not in pad_groups]
    qv = q.view(-1, P, 4)
    qb = []
    for (g, n, end), dst in zip(qblocks[1:], live):
        qp[dst] = qv[g]
        qb.append((dst, n, end))
    for g in pad_groups:
        qp[g] = 0
        qb.append((g, 0, P))
    inp['geo_memory_points'] = mem.view(B, N, 11).contiguous()
    inp['geo_query_points'] = qp.view(B, Q, P, 4).contiguous()
    inp['geo_query_num'] = num
    return inp, mblocks, qb


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_tied_rows_give_the_same_gradients(mode):
    """through the module: each tie group pools at its block's first row (m.reg.pooled_rows), and the step's gradients match the
    float64 restatement pooled at the lowest, the highest and a random row of each tie set (the three restatements agree among
    themselves to float64 rounding): the point layers' gradients within the step bounds in both modes, the point paths' outputs
    within the forward bound, and the other gradients within the step bounds of float64 restated from those outputs (in fp32 of
    the full restatement too)"""
    seed = SEED + 9
    inp, mblocks, qblocks = tie_inputs(seed)
    m = grm(mode, seed)
    sd = clone_sd(m)
    _, _, _, grads, _ = step(m, inp)
    rows = {k: v.cpu() for k, v in m.reg.pooled_rows.items()}
    check_block_rows(rows['memory'].long().unsqueeze(0), mblocks, 4096, 4096 - 56, 'memory')
    check_block_rows(rows['query'].long().unsqueeze(0), qblocks, 256, 256 - 56, 'query')
    rec = {}
    grm_train_ref.grm_train_step(sd, inp, device='cuda', pooled_rows=rows, record=rec)
    alt = {}
    for how in ('lowest', 'highest', 'random'):
        r = {}
        for k in ('memory', 'query'):
            y = rec[k].cpu()                                         # (groups, rows, C)
            P = y.shape[1]
            dev_val = y.gather(1, rows[k].long().unsqueeze(1))
            tie = y == dev_val                                       # the tie set of the device's row
            pr = torch.arange(P).view(1, P, 1).expand_as(y)
            if how == 'lowest':
                r[k] = torch.where(tie, pr, P).min(1)[0]
                pos = dev_val.squeeze(1) > 0                             # the device pools at the lowest row of a positive tie
                assert torch.equal(r[k].int()[pos], rows[k][pos]), k
            elif how == 'highest':
                r[k] = torch.where(tie, pr, -1).max(1)[0]
            else:
                key = torch.rand(y.shape, generator=torch.Generator().manual_seed(3)) + tie.double()
                r[k] = key.max(1)[1]
        alt[how] = grm_train_ref.grm_train_step(sd, inp, device='cuda', pooled_rows=r)[1]
    floor = FLOOR * max(g.abs().max().item() for g in alt['lowest'].values())
    for how in ('highest', 'random'):
        for k, g in alt[how].items():
            assert err(g, alt['lowest'][k], floor) <= 1e-10, (how, k)
    # the point layers' gradients against the restatement in both modes; the rest of the step (query MLP, decoder, heads: torch
    # autograd on the device) against float64 restated from the device's own point-path outputs, which are held to the forward
    # bound first.  Measured in tf32 on an H100 80GB HBM3: the device's pooled memory output is 5e-4 off float64 (TF32 autograd
    # 6e-4), yet the decoder and head gradients end to end are up to 2e-1 off (TF32 autograd 2e-2).  Restating layer 5 at the
    # device's own ReLU masks changes none of it, and the point layers' own gradients are within the bounds, so the excess arises
    # downstream, from rounding-sized differences in the point-path outputs; the end-to-end comparison in tf32 would measure that
    # sensitivity of these inputs, not the kernels.  In fp32 the end-to-end comparison holds as well.
    point = ('memory_encoder.', 'memory_mlp.', 'query_encoder.')
    ref_err = lambda k, g: err(g, alt['lowest'][k], floor)          # noqa: E731
    ag = autograd_errors(sd, inp, mode, ref_err, rows, floor)
    held = grads if mode == 'fp32' else {k: g for k, g in grads.items() if k.startswith(point)}
    bad = {k: (ref_err(k, g), ag[k]) for k, g in held.items() if ref_err(k, g) > max(TOL[mode]['grad'], ASSOC * ag[k])}
    assert not bad, bad
    with torch.no_grad():
        m2 = grm(mode, seed)
        outs = {'memory_out': train.grm_memory(m2.reg, inp['geo_memory_points'].float()),
                'query_pool': train.grm_query(m2.reg, inp['geo_query_points'].float())}
    assert torch.equal(m2.reg.pooled_rows['memory'].cpu(), rows['memory'])
    rec32 = autograd_record(sd, inp, mode, rows)
    for k in ('memory_out', 'query_pool'):
        assert path_err(outs[k], rec[k]) <= max(TOL[mode]['stats'], ASSOC * path_err(rec32[k], rec[k])), k
    _, dgrads, _ = grm_train_ref.grm_train_step(sd, inp, device='cuda', pooled_rows=rows, path_outputs=outs)
    assert not any(k.startswith(point) for k in dgrads)
    dfloor = FLOOR * max(g.abs().max().item() for g in dgrads.values())
    derr = {k: err(grads[k], g, dfloor) for k, g in dgrads.items()}
    assert max(derr.values()) <= TOL[mode]['grad'], sorted(derr.items(), key=lambda kv: -kv[1])[:4]


# ---- a step on samples built from a tracked sequence ------------------------------------------------------------------------
def _targets(s, seed=2):
    """TrackTargets of a synthetic sequence: ground truth near each box, some unmatched slots, every track a matched tracklet with a
    matched box"""
    g = np.random.default_rng(seed)
    B, L = s['boxes'].shape[:2]
    valid = np.arange(L)[None, :] < np.asarray(s['box_num'])[:, None]
    matched = valid & (g.random((B, L)) < 0.8)
    matched[:, 0] |= valid[:, 0]
    gt = s['boxes'] + np.concatenate([g.normal(0, 0.1, (B, L, 3)), g.normal(0, 0.05, (B, L, 3)), g.normal(0, 0.02, (B, L, 1))], 2)
    gt[~matched] = 0
    t = lambda a, dt: torch.as_tensor(a, dtype=dt, device='cuda')  # noqa: E731
    return rdata.TrackTargets(t(gt, torch.float64), t(matched, torch.uint8), t(np.ones(B), torch.uint8), t(np.ones(B), torch.int32),
                              t(np.zeros((B, L, 7)), torch.float32), t(np.arange(B), torch.int32))


def built_inputs():
    """a GRM batch built on the device by geometry_training_inputs from a tracked synthetic sequence: tracks of 1 and 2 boxes (their
    padded queries are all zero), boxes with no point and with a few (their memory samples repeat one encoded point)"""
    s = synthetic.synthetic_sequence(3, frames=24, tracks=10, n_background=20000, lengths=[24, 1, 2, 17, 24, 5, 9, 24, 3, 12])
    dev = torch.device('cuda')
    tb = rdata.TrackBatch(s['boxes'], s['frame_of_box'], s['scores'], s['box_num'], s['cls'], s['track_uid'], dev)
    out = rdata.geometry_training_inputs(torch.from_numpy(s['frames']).to(dev), s['frame_offsets'], torch.from_numpy(s['poses']).to(dev),
                                         tb, _targets(s), seed=SEED, epoch=3, return_selection=True)
    num = out['geo_query_num'].cpu()
    Q = out['geo_query_points'].shape[1]
    kn = out['kept_num'].cpu()
    assert (kn == 1).any() and (kn == 2).any() and (num < Q).any(), (kn, num)
    pad = torch.arange(Q)[None] >= num[:, None]
    assert (out['geo_query_points'].cpu()[pad] == 0).all()
    kept = out['kept'].cpu() >= 0
    counts = out['crop_counts'].cpu()[kept]
    assert (counts == 0).any() and ((counts > 0) & (counts < 16)).any() and (counts > 256).any(), counts
    return {k: out[k] for k in ('geo_memory_points', 'geo_query_points', 'geo_query_boxes', 'geo_query_num', 'gt_geo_query_boxes')}


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_step_on_built_samples_at_device_pooled_rows(mode):
    """the device step on built samples against the float64 restatement pooled at the device's rows: losses, every gradient, the
    running statistics, and the pooled memory output g, the memory path's output and the pooled query output element by element;
    every pooled row within the
    forward bound of the float64 maximum, and no more flips than float32 autograd"""
    tol = TOL[mode]
    inp = built_inputs()
    seed = SEED + 5
    m = grm(mode, seed)
    sd = clone_sd(m)
    _, tb, _, grads, stats = step(m, inp)
    rows = {k: v.cpu() for k, v in m.reg.pooled_rows.items()}
    with torch.no_grad():
        m2 = grm(mode, seed)
        mem = train.grm_memory(m2.reg, inp['geo_memory_points'].float())
        qpool = train.grm_query(m2.reg, inp['geo_query_points'].float())
    for k in rows:
        assert torch.equal(m2.reg.pooled_rows[k].cpu(), rows[k]), k
    rec = {}
    losses, rgrads, rstats = grm_train_ref.grm_train_step(sd, inp, device='cuda', pooled_rows=rows, record=rec)
    for k, v in losses.items():
        assert abs(tb[k].item() - v) <= tol['loss'] * abs(v), (k, tb[k].item(), v)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = mode == 'tf32'
    rec32 = {}
    try:
        _, g32, _ = grm_train_ref.grm_train_step(sd, inp, device='cuda', pooled_rows=rows, dtype=torch.float32, record=rec32)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    # each output channel against its largest value over the rows; allowed ASSOC times the error of float32 autograd at the same rows:
    # the pooled memory output g, the memory path's output and the pooled query output
    for k, got in (('memory_pool', rows['memory_pool']), ('memory_out', mem), ('query_pool', qpool)):
        e, e32 = path_err(got, rec[k]), path_err(rec32[k], rec[k])
        assert e <= max(tol['stats'], ASSOC * e32), (k, e, e32)
    floor = FLOOR * max(g.abs().max().item() for g in rgrads.values())
    errs = {k: err(g, rgrads[k], floor) for k, g in grads.items()}
    ag = {k: err(g, rgrads[k], floor) for k, g in g32.items()}
    bad = {k: (e, ag[k]) for k, e in errs.items() if e > max(tol['grad'], ASSOC * ag[k])}
    assert not bad, bad
    check_stats(stats, rstats, tol['stats'])
    check_pooled_rows(m, sd, inp, mode)


# ---- what the C ABI refuses, before it enqueues anything ---------------------------------------------------------------------
def test_c_abi_rejections_leave_outputs_untouched():
    """R or gsize not a multiple of 64, a gsize that does not divide R, forward N / dgrad Kout not a multiple of 128, a dgrad
    segment N not a multiple of 32, wgrad N not a multiple of 64, nseg not 1 or 2, a pooled segment with sel but no dsel, and a mode
    other than fp32 / tf32 each return their code, and the output buffers keep their contents"""
    L, P, st = _lib.lib(), ops._p, ops._stream
    UNS, ARG = -4, -1
    dev = 'cuda'
    R, K, N = 512, 128, 256
    x = torch.randn(R, K, device=dev)
    w = torch.randn(N, K, device=dev)
    wt = torch.randn(K, N, device=dev)
    tk, tn = table(K, torch.Generator(device=dev).manual_seed(1), dev), table(N, torch.Generator(device=dev).manual_seed(2), dev)
    zn = torch.randn(R, N, device=dev)
    sel = torch.zeros(R // 128, N, dtype=torch.int32, device=dev)
    outs = {'z': torch.full((R, N), 7.0, device=dev), 'ps': torch.full((R // 64, 2, max(N, K)), 7.0, dtype=torch.float64, device=dev),
            'ev': torch.full((R // 64, 2, N), 7.0, device=dev), 'ei': torch.full((R // 64, 2, N), 7, dtype=torch.int32, device=dev),
            'dh': torch.full((R, K), 7.0, device=dev), 'dw': torch.full((N, K), 7.0, dtype=torch.float64, device=dev)}
    before = {k: v.clone() for k, v in outs.items()}
    ws = torch.empty(L.dz_pm_wgrad_ws_bytes(R, N, K) + (1 << 20), dtype=torch.uint8, device=dev)

    def fwd(mode=1, R=R, gsize=128, N=N):
        return L.dz_pm_fwd(mode, P(x), R, K, P(tk), P(w), N, P(None), gsize, P(outs['z']), P(outs['ps']), P(outs['ev']), P(outs['ei']),
                           st())

    def dgrad(mode=1, R=R, gsize=128, nseg=1, N1=N, Kout=K, dh1=zn, sel1=None, dsel1=None):
        return L.dz_pm_dgrad(mode, R, gsize, nseg, N1, P(dh1), P(sel1), P(dsel1), P(zn), P(tn), P(wt),
                             N, P(zn), P(None), P(None), P(zn), P(tn), P(wt), Kout, P(x), P(tk), P(outs['dh']), P(outs['ps']), st())

    def wgrad(mode=1, R=R, gsize=128, N=N, dh=zn, sel=None, dsel=None):
        return L.dz_pm_wgrad(mode, R, gsize, N, P(dh), P(sel), P(dsel), P(zn), P(tn), P(x), K, P(tk), P(outs['dw']), P(ws), ws.numel(),
                             st())

    def dh(R=R):
        return L.dz_pm_dh(R, N, P(zn), P(zn), P(tn), P(outs['z']), P(outs['ps']), st())

    cases = [(fwd(R=R - 32), UNS), (fwd(gsize=96), UNS), (fwd(gsize=192), UNS), (fwd(N=192), UNS), (fwd(mode=2), UNS),
             (fwd(mode=-1), UNS),
             (dgrad(R=R - 32), UNS), (dgrad(gsize=96), UNS), (dgrad(gsize=192), UNS), (dgrad(Kout=64), UNS), (dgrad(N1=48), UNS),
             (dgrad(nseg=0), ARG), (dgrad(nseg=3), ARG), (dgrad(dh1=None, sel1=sel), ARG), (dgrad(mode=2), UNS),
             (wgrad(R=R - 32), UNS), (wgrad(gsize=96), UNS), (wgrad(gsize=192), UNS), (wgrad(N=96), UNS),
             (wgrad(dh=None, sel=sel), ARG), (wgrad(mode=3), UNS),
             (dh(R=R - 32), UNS), (dh(R=100), UNS)]
    for i, (rc, want) in enumerate(cases):
        assert rc == want, (i, rc, want, L.dz_last_error_string())
    torch.cuda.synchronize()
    for k, v in outs.items():
        assert torch.equal(v, before[k]), k
    # the same arguments with the offending one corrected are accepted
    assert fwd() == 0 and dgrad() == 0 and wgrad() == 0 and dh() == 0
    torch.cuda.synchronize()

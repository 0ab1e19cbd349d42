"""Element-wise checks of the refiner kernels -- dz_linear_fwd(_grouped), dz_linear_max_fwd, dz_group_max, dz_attention_fwd and
dz_layernorm_residual, in the exact-fp32 and the TF32 tensor-core modes -- against float64 torch restatements of the same
operations, at the shapes the config-4 refiner (PRM / GRM / CRM) runs and at the tile and key-block edges of the kernels.

Every bound is derived from operand rounding, not fitted to observed errors.  u = 2^-24 is the fp32 unit roundoff.  The tensor core
reads an fp32 operand with its low 13 mantissa bits dropped (TF32), a relative error below 2^-10 for an operand that is not already
TF32-representable; its products of two TF32 values are exact in fp32 and only its adder rounds.  Where a bound is a maximum over
rows of a column (group max), |max a - max b| <= max |a - b| carries the per-row bound over.  Every failure reports the largest
err / bound ratio and where it occurs."""
import inspect

import numpy as np
import pytest
import torch

from detzero_b200 import _lib, ops, synthetic
from tests.util import assert_equal_signed as _assert_equal_signed, assert_within as _assert_within

pytestmark = pytest.mark.gpu
F64 = torch.float64
U = 2.0 ** -24               # fp32 unit roundoff
TF32_READ = 2.0 ** -10       # relative error of the tensor core's truncating read of an fp32 operand
TF32_HALF_ULP = 2.0 ** -11   # cvt.rna.tf32 of a ReLU output (the TF32 linear epilogue rounds what feeds the next TF32 layer)
TC_ADD = 16                  # safety factor on the tensor-core adder: K products accumulate with <= 16 K u |terms| of error
F32, TF32 = _lib.DZ_F32, _lib.DZ_TF32
MODES = {'fp32': F32, 'tf32': TF32}


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _tf32_exact(t):
    return torch.equal(t, ops.round_tf32(t))



# ---------------------------------------------------------------------------------------------------------------------------------
# linear layers: y = act((x W^T) * scale + shift [+ gshift[row // gsize]])
# ---------------------------------------------------------------------------------------------------------------------------------
def _linear_ref(x, w, scale, shift, relu, mode, gshift=None, gsize=1, rows=None):
    """float64 reference of the rows `rows` of x (all rows if None) and the bound before any output rounding.

    fp32 kernel (FMA chain over K, then one multiply and up to two adds, each rounded):
        |y - y64| <= (K + 3) u (|scale| A + |shift| + |gshift|),     A = |x| @ |w|^T
    TF32 kernel: the same epilogue, the tensor-core adder (TC_ADD K u |scale| A), and 2^-10 |scale| A for each operand (x, W) that is
    not TF32-representable.  ReLU is 1-Lipschitz, so it keeps the bound; the output rounding of a TF32 ReLU layer is added by the
    caller (it depends on the output)."""
    K = x.shape[1]
    x64 = (x if rows is None else x[rows]).to(F64)
    w64 = w.to(F64)
    y, A = x64 @ w64.t(), x64.abs() @ w64.abs().t()
    sa = A
    if scale is not None:
        y, sa = y * scale.to(F64), A * scale.to(F64).abs()
    c = torch.zeros_like(y)
    if shift is not None:
        y, c = y + shift.to(F64), c + shift.to(F64).abs()
    if gshift is not None:
        r = torch.arange(x.shape[0], device=x.device) if rows is None else rows.to(x.device)
        g = gshift.to(F64)[r // gsize]
        y, c = y + g, c + g.abs()
    if relu:
        y = y.clamp_min(0)
    bound = (K + 3) * U * (sa + c)
    if mode == TF32:
        bound = bound + TC_ADD * K * U * sa
        reads = (0 if _tf32_exact(x if rows is None else x[rows]) else 1) + (0 if _tf32_exact(w) else 1)
        bound = bound + reads * TF32_READ * sa
    return y, bound


def _check_linear(out, x, w, scale, shift, relu, mode, what, gshift=None, gsize=1, rows=None):
    y64, bound = _linear_ref(x, w, scale, shift, relu, mode, gshift, gsize, rows)
    got = out if rows is None else out[rows.to(out.device)]
    if mode == TF32 and relu:
        bound = bound + TF32_HALF_ULP * got.to(F64).abs()
    return _assert_within(got, y64, bound, what)


def _rand_linear(g, M, K, N, has_scale, has_shift, dev, tf32_x=False):
    x = torch.randn(M, K, generator=g)
    if tf32_x:
        x = ops.round_tf32(x)
    w = torch.randn(N, K, generator=g) * K ** -0.5
    scale = (torch.rand(N, generator=g) + 0.5) * torch.where(torch.rand(N, generator=g) < 0.2, -1.0, 1.0) if has_scale else None
    shift = torch.randn(N, generator=g) if has_shift else None
    mv = lambda t: None if t is None else t.to(dev)          # noqa: E731
    return x.to(dev), w.to(dev), mv(scale), mv(shift)


def _weights(w, mode):
    return ops.round_tf32(w) if mode == TF32 else w


def _sample_rows(M, block, budget=1 << 16):
    """all rows, or whole blocks of `block` rows -- the first, the last, evenly spread ones between -- plus the rows past the last
    whole block (the M % 16 tail of a TF32 linear is among them)"""
    if M <= budget:
        return torch.arange(M)
    nb = M // block
    k = max(2, min(34, budget // block))
    starts = sorted(set(np.linspace(0, nb - 1, k).round().astype(int).tolist()))
    return torch.cat([torch.arange(s * block, (s + 1) * block) for s in starts] + [torch.arange(nb * block, M)])


# ---- the refiner modules at the config-4 shapes, with the GEMM-like ops wrapped ------------------------------------------------
def _config4_forwards(dev, mode):
    """one forward each of PRM (16 tracks x 200 boxes x 1024 query points), GRM (16 tracks, 4096 memory points) and CRM (16 x 200 x 256)"""
    from detzero_b200.refine import ConfidencePointnet, GeometryTransformer, PositionTransformer
    runs = ((PositionTransformer, synthetic.prm_cfg, (32, 32), 4321, synthetic.prm_inputs(100, B=16, qpts=1024)),
            (GeometryTransformer, synthetic.grm_cfg, (11, 4), 4322, synthetic.grm_inputs(200, B=16)),
            (ConfidencePointnet, synthetic.crm_cfg, (32, 32), 4323, synthetic.crm_inputs(300, B=16)))
    for cls, cfg_fn, dims, seed, inputs in runs:
        cfg = cfg_fn()
        cfg.COMPUTE_MODE = {F32: 'fp32', TF32: 'tf32'}[mode]
        m = cls(cfg, *dims).eval()
        synthetic.load_seeded(m, seed)
        m = m.to(dev)
        with torch.no_grad():
            m({k: v.to(dev) if isinstance(v, torch.Tensor) else v for k, v in inputs.items()})
        del m
    torch.cuda.synchronize()


def _wrap(mp, name, after):
    """replace ops.<name> by a wrapper that calls the kernel and then after(bound arguments, result)"""
    orig = getattr(ops, name)
    sig = inspect.signature(orig)

    def wrapper(*args, **kwargs):
        out = orig(*args, **kwargs)
        a = sig.bind(*args, **kwargs)
        a.apply_defaults()
        after(a.arguments, out)
        return out
    mp.setattr(ops, name, wrapper)


@pytest.fixture(scope='module')
def config4_linear_shapes(cuda):
    """(K, N) of every ops.linear call of the config-4 refiner modules, in both modes"""
    shapes = set()
    with pytest.MonkeyPatch.context() as mp:
        _wrap(mp, 'linear', lambda a, out: shapes.add((a['x'].shape[1], a['w'].shape[0])))
        for mode in (F32, TF32):
            _config4_forwards(cuda, mode)
    return sorted(shapes)


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_config4_calls_elementwise(cuda, mode, monkeypatch):
    """every linear / grouped linear / fused linear+max / group max the PRM, GRM and CRM forwards issue, on their real operands
    (rows / groups sampled where the float64 reference would not fit in a few hundred MB)"""
    mode = MODES[mode]
    seen = {}

    def linear(a, out):
        x, w = a['x'], a['w']
        key = ('linear', x.shape[0], x.shape[1], w.shape[0], a['scale'] is not None, a['shift'] is not None, bool(a['relu']))
        seen[key] = seen.get(key, 0) + 1
        rows = _sample_rows(x.shape[0], 1024).to(x.device)
        _check_linear(out, x, w, a['scale'], a['shift'], a['relu'], a['mode'], 'linear %s' % (key[1:],), rows=rows)

    def grouped(a, out):
        x, w, gsize = a['x'], a['w'], a['gsize']
        key = ('linear_grouped', x.shape[0], x.shape[1], w.shape[0], gsize, bool(a['relu']))
        seen[key] = seen.get(key, 0) + 1
        rows = _sample_rows(x.shape[0], gsize).to(x.device)
        _check_linear(out, x, w, a['scale'], a['shift'], a['relu'], a['mode'], 'linear_grouped %s' % (key[1:],),
                      gshift=a['gshift'], gsize=gsize, rows=rows)

    def linear_max(a, out):
        x, w, group = a['x'], a['w'], a['group']
        key = ('linear_max', x.shape[0], x.shape[1], w.shape[0], group, bool(a['relu']))
        seen[key] = seen.get(key, 0) + 1
        G = x.shape[0] // group
        gs = torch.from_numpy(np.unique(np.linspace(0, G - 1, max(2, min(34, (1 << 16) // group))).round().astype(int)))
        rows = (gs[:, None] * group + torch.arange(group)[None, :]).reshape(-1).to(x.device)
        y64, bound = _linear_ref(x, w, a['scale'], a['shift'], a['relu'], a['mode'], rows=rows)
        n = w.shape[0]
        _assert_within(out[gs.to(out.device)], y64.view(-1, group, n).amax(1), bound.view(-1, group, n).amax(1),
                       'linear_max %s' % (key[1:],))

    def group_max(a, out):
        x, G, group = a['x'], a['G'], a['group']
        seen[('group_max', G, group, x.shape[1])] = 1
        _assert_equal_signed(out, x.view(G, group, -1).amax(1), 'group_max G=%d group=%d' % (G, group))

    _wrap(monkeypatch, 'linear', linear)
    _wrap(monkeypatch, 'linear_grouped', grouped)
    _wrap(monkeypatch, 'linear_max', linear_max)
    _wrap(monkeypatch, 'group_max', group_max)
    _config4_forwards(cuda, mode)
    kinds = {k[0] for k in seen}
    assert {'linear', 'linear_grouped', 'group_max'} <= kinds and (mode == F32 or 'linear_max' in kinds), kinds
    assert any(k[0] == 'linear' and k[2] in (3, 4, 11) for k in seen)          # the K < 32 layers on the fp32 fallback
    assert any(k[0] == 'linear' and k[3] == 768 for k in seen)                 # the packed qkv projection


def test_tf32_weight_operands_are_rounded(cuda, monkeypatch):
    """in TF32 mode every weight that reaches a tensor-core GEMM is RN-rounded to TF32 beforehand (ops.round_tf32): the tensor core
    truncates the fp32 container, and truncated weights bias every output toward zero"""
    bad = []

    def rec(name):
        def after(a, out):
            w = a['w']
            if not _tf32_exact(w):
                bad.append((name, tuple(w.shape)))
        return after
    for name in ('linear', 'linear_grouped', 'linear_max'):
        _wrap(monkeypatch, name, rec(name))
    _config4_forwards(cuda, TF32)
    assert not bad, 'weights not rounded to TF32: %s' % sorted(set(bad))


@pytest.mark.parametrize('variant', ['fp32', 'tf32', 'tf32_exact_x'])
def test_linear_shapes(cuda, config4_linear_shapes, variant):
    """every (K, N) of the config-4 modules x M in {1, 15, 16, 17, 129, 3200} (the TF32 path below 16 rows, at one 16-row block, with
    tail rows, across 128-row tiles) x scale / shift present or not x ReLU on / off; plus the ragged channel tiles N = 36, 100.
    tf32_exact_x feeds TF32-representable activations: only the accumulation is left, which leaves no room for a dropped k8 step
    (~ 8 / K |y|)"""
    mode = F32 if variant == 'fp32' else TF32
    g = _gen(11)
    shapes = sorted(set(config4_linear_shapes) | {(32, 36), (128, 100), (4, 36)})
    assert any(K in (3, 4, 11, 32) for K, _ in shapes) and any(N in (3, 9, 12) for _, N in shapes) and any(N == 768 for _, N in shapes)
    for K, N in shapes:
        for M in (1, 15, 16, 17, 129, 3200):
            for flags in range(8):
                has_scale, has_shift, relu = bool(flags & 1), bool(flags & 2), bool(flags & 4)
                x, w, sc, sh = _rand_linear(g, M, K, N, has_scale, has_shift, cuda, tf32_x=variant == 'tf32_exact_x')
                w = _weights(w, mode)
                out = ops.linear(x, w, sc, sh, relu, mode=mode)
                _check_linear(out, x, w, sc, sh, relu, mode, '%s linear M=%d K=%d N=%d scale=%d shift=%d relu=%d'
                              % (variant, M, K, N, has_scale, has_shift, relu))


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_linear_into_wider_output(cuda, mode):
    """ldy > N: the layer writes columns [c0, c0 + N) of a wider, sentinel-filled buffer and nothing else"""
    mode = MODES[mode]
    g = _gen(12)
    for M, K, N, c0, ldy in ((129, 32, 36, 4, 44), (3200, 128, 100, 4, 108), (17, 128, 12, 0, 17), (1000, 256, 256, 0, 260)):
        x, w, sc, sh = _rand_linear(g, M, K, N, True, True, cuda)
        w = _weights(w, mode)
        buf = torch.full((M, ldy), -7.25e30, device=cuda)
        out = ops.linear(x, w, sc, sh, True, out=buf[:, c0:c0 + N], mode=mode)
        _check_linear(out, x, w, sc, sh, True, mode, 'linear M=%d N=%d into ldy=%d at column %d' % (M, N, ldy, c0))
        outside = torch.cat([buf[:, :c0], buf[:, c0 + N:]], dim=1)
        assert bool((outside == -7.25e30).all()), 'linear M=%d N=%d ldy=%d wrote outside its columns' % (M, N, ldy)


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_linear_grouped(cuda, mode):
    """y[m] = act((x[m] W^T) * scale + shift + gshift[m // gsize]): the rows past the last 16-row block of the TF32 path go through the
    fp32 kernel with a row offset, and must still pick their own group.  gsize 9 and 200 with an odd group count leave such tail rows
    (M % 16 = 11, 8); 16, 48 and 9600 are multiples of 16 and never do"""
    mode = MODES[mode]
    g = _gen(13)
    for gsize, G, K, N in ((9, 3, 128, 36), (16, 5, 128, 512), (48, 7, 128, 512), (200, 5, 128, 256), (200, 1, 32, 12), (9600, 2, 128, 512)):
        M = G * gsize
        x, w, sc, sh = _rand_linear(g, M, K, N, True, True, cuda)
        w = _weights(w, mode)
        gshift = (torch.randn(G, N, generator=g) * 3).to(cuda)
        for relu in (False, True):
            out = ops.linear_grouped(x, w, gshift, gsize, sc, sh, relu, mode=mode)
            _check_linear(out, x, w, sc, sh, relu, mode, 'linear_grouped gsize=%d G=%d relu=%d' % (gsize, G, relu), gshift=gshift, gsize=gsize)


def _linear_max_ref(x, w, group, sc, sh, relu):
    y64, bound = _linear_ref(x, w, sc, sh, relu, TF32)         # the fused epilogue does not round its ReLU output
    n = w.shape[0]
    return y64.view(-1, group, n).amax(1), bound.view(-1, group, n).amax(1)


def test_linear_max(cuda):
    """fused last PointNet layer + max over groups of `group` rows (TF32 only): groups of one 128-row tile to 75 tiles, N = 4 (one
    narrow channel tile), 36 (ragged), 256; ReLU on and off"""
    g = _gen(14)
    for group, G in ((128, 37), (256, 16), (1024, 5), (4096, 3), (9600, 2)):
        for N in (4, 36, 256):
            for relu in (True, False):
                x, w, sc, sh = _rand_linear(g, G * group, 128, N, True, True, cuda)
                w = ops.round_tf32(w)
                out = ops.linear_max(x, w, group, sc, sh, relu, mode=TF32)
                ref, bound = _linear_max_ref(x, w, group, sc, sh, relu)
                _assert_within(out, ref, bound, 'linear_max group=%d N=%d relu=%d' % (group, N, relu))


def test_linear_max_negative_and_signed_zero(cuda):
    """relu=False with every output negative (every group maximum through the negative-float atomic), and groups whose maximum is
    exactly -0.0: all-zero rows times a negative folded-BN scale with no shift give -0.0, which torch.max returns"""
    g = _gen(15)
    group, G, K, N = 256, 6, 64, 36
    x = torch.rand(G * group, K, generator=g) + 0.1
    w = ops.round_tf32(torch.rand(N, K, generator=g) * K ** -0.5 + 0.01)
    sc = -(torch.rand(N, generator=g) + 0.5)
    sh = -torch.rand(N, generator=g)
    x, w, sc, sh = x.to(cuda), w.to(cuda), sc.to(cuda), sh.to(cuda)
    out = ops.linear_max(x, w, group, sc, sh, False, mode=TF32)
    ref, bound = _linear_max_ref(x, w, group, sc, sh, False)
    assert bool((ref < 0).all())
    _assert_within(out, ref, bound, 'linear_max all-negative')
    # group 0: every row zero; group 1: zero rows among positive ones (the maximum is still -0.0); no shift
    x[:group] = 0
    x[group + 17:group + 20] = 0
    out = ops.linear_max(x, w, group, sc, None, False, mode=TF32)
    ref, bound = _linear_max_ref(x, w, group, sc, None, False)
    assert bool((ref[:2] == 0).all() and torch.signbit(ref[:2]).all())
    _assert_within(out, ref, bound, 'linear_max with -0.0 maxima')
    _assert_equal_signed(out[:2], ref[:2], 'linear_max -0.0 group maxima')


# ---------------------------------------------------------------------------------------------------------------------------------
# group max: exact, compared bit for bit (sign of zero included)
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('G,group,C,branch', [
    (16, 9600, 256, 'split'),        # the PRM memory pool: G*C < 75776 and group >= 256: rows split over CTAs, atomic max
    (16, 4096, 128, 'split'),
    (3, 300, 36, 'split'),           # a partial 64-row slice at the end of each group, C < 128
    (3200, 256, 256, 'column'),      # one thread per (group, column)
    (16, 200, 256, 'column'),        # group < 256
    (1000, 1, 100, 'column'),        # group = 1: a copy
])
def test_group_max(cuda, G, group, C, branch):
    g = _gen(G * 7 + group)
    x = torch.randn(G * group, C, generator=g)
    x3 = x.view(G, group, C)
    x3[0] = -x3[0].abs() - 0.5                                   # a group with only negative values
    if G > 1 and group > 1:
        x3[1] = -x3[1].abs()                                     # ... whose maximum is -0.0
        x3[1, group // 2, :] = -0.0
        x3[1, -1, : C // 2] = -0.0                               # twice in some columns, in the last rows of the group
    elif G > 1:
        x3[1] = -0.0
    y = ops.group_max(x.to(cuda), G, group)
    _assert_equal_signed(y, x3.amax(1), 'group_max %s G=%d group=%d C=%d' % (branch, G, group, C))


# ---------------------------------------------------------------------------------------------------------------------------------
# attention: softmax(q k^T + mask) v per (batch, head), head_dim 32
# ---------------------------------------------------------------------------------------------------------------------------------
def _attention_ref(q, k, v, mask, H, mode):
    """float64 softmax(q k^T, masked keys -> -inf) v (NaN rows where every key is masked, as torch) and its bound, per (b, h).

    Logit error: fp32, an FMA chain over dh: ds_j <= 2 dh u S_j with S = |q| @ |k|^T; TF32: the tensor-core adder TC_ADD dh u S_j, plus
    2 * 2^-10 S_j for the truncating reads of q and k unless both are TF32-representable.  The exponent's argument s - m is
    formed in fp32: + 4 u (|s_j| + |m|).  If every unnormalised weight is off by a factor e^{e_j}, |e_j| <= D, the normalised weights
    are off by at most e^{2D}, so |o - o64| <= expm1(2 D) sum_j p_j |v_j|, D = max over valid keys of ds_j.
    The weighted sum itself: fp32, <= Pk / 2 + Pk / 64 sequential FMAs / rescales per output and the final 1 / l:
    (2 Pk + 16) u sum_j p_j |v_j|; TF32, P is truncated to TF32 (2^-10) and so is V unless representable, and the registers
    accumulate Pk products (<= 4 u each, with the row sum l) and ex2.approx: (2^-10 [+ 2^-10] + (5 Pk + 32) u) sum_j p_j |v_j|."""
    B, Pq, E = q.shape
    Pk, dh = k.shape[1], E // H
    qk_reads = 0 if _tf32_exact(q) and _tf32_exact(k) else 2
    v_reads = 0 if _tf32_exact(v) else 1
    ref = torch.empty(B, Pq, E, dtype=F64, device=q.device)
    bound = torch.empty_like(ref)
    for b in range(B):
        valid = torch.ones(Pk, dtype=torch.bool, device=q.device) if mask is None else mask[b] == 0
        for h in range(H):
            sl = slice(h * dh, (h + 1) * dh)
            qh, kh, vh = q[b, :, sl].to(F64), k[b, :, sl].to(F64), v[b, :, sl].to(F64)
            s = (qh @ kh.t()).masked_fill(~valid, float('-inf'))
            S = qh.abs() @ kh.abs().t()
            p = torch.softmax(s, dim=-1)
            ref[b, :, sl] = p @ vh
            if mode == F32:
                ds = 2 * dh * U * S
                c = (2 * Pk + 16) * U
            else:
                ds = (TC_ADD * dh * U + qk_reads * TF32_READ) * S
                c = (1 + v_reads) * TF32_READ + (5 * Pk + 32) * U
            m = s.amax(dim=-1, keepdim=True)
            ds = (ds + 4 * U * (s.abs() + m.abs())).masked_fill(~valid, 0).amax(dim=-1, keepdim=True)
            bound[b, :, sl] = (torch.expm1(2 * ds) + c) * (p @ vh.abs())
    return ref, bound


def _check_attention(q, k, v, mask, H, mode, what):
    out = ops.attention(q, k, v, mask, H, mode=mode)
    ref, bound = _attention_ref(q, k, v, mask, H, mode)
    return _assert_within(out, ref, bound, what)


def _randn_tf32(g, *shape, scale=1.0):
    """TF32-representable operands: the TF32 kernel reads them exactly, which leaves a bound ~30x sharper than for arbitrary fp32"""
    return ops.round_tf32(torch.randn(*shape, generator=g) * scale)


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
@pytest.mark.parametrize('layout', ['prm_self', 'prm_cross', 'grm_cross'])
def test_attention_production_layouts(cuda, mode, layout):
    """q / k / v exactly as MultiheadAttention.forward_tokens makes them: strided column slices of the packed projection
    (self-attention: row stride 3E = 768; cross-attention: q contiguous, k / v row stride 2E = 512), with the masks PositionHead builds
    (self: the box padding mask; cross: the padding mask repeated over the 48 memory points of a box); GRM cross-attention: 3 queries
    against 4096 memory points, no mask.  Once with arbitrary fp32 operands, once with TF32-representable ones (sharper bound)"""
    mode = MODES[mode]
    g = _gen(21)
    B, E, H = 16, 256, 8
    scale = (E // H) ** -0.5
    pad = synthetic.prm_inputs(100, B=B)['padding_mask'] != 0
    for rnd in (lambda t: t, ops.round_tf32):
        if layout == 'prm_self':
            qkv = torch.randn(B, 200, 3 * E, generator=g)
            qkv[..., :E] *= scale
            qkv = rnd(qkv).to(cuda)
            q, k, v = qkv[:, :, :E], qkv[:, :, E:2 * E], qkv[:, :, 2 * E:]
            mask = pad.to(torch.uint8).contiguous().to(cuda)
        else:
            Pq, Pk = (200, 200 * 48) if layout == 'prm_cross' else (3, 4096)
            q = rnd(torch.randn(B, Pq, E, generator=g) * scale).to(cuda)
            kv = rnd(torch.randn(B, Pk, 2 * E, generator=g)).to(cuda)
            k, v = kv[:, :, :E], kv[:, :, E:]
            mask = None
            if layout == 'prm_cross':
                mask = pad.to(torch.uint8).view(B, 200, 1).expand(B, 200, 48).reshape(B, -1).contiguous().to(cuda)
        _check_attention(q, k, v, mask, H, mode, 'attention %s%s' % (layout, '' if rnd is not ops.round_tf32 else ', TF32-representable'))


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
@pytest.mark.parametrize('H', [1, 8])
def test_attention_block_edges(cuda, mode, H):
    """Pq around the 64 / 128-query tiles x Pk around the 64 / 128-key blocks; B = 2, so the Q and K boxes of the last batch run past
    the end of the tensor and those of the first batch into the second; batch 0 masks a third of its keys at random"""
    mode = MODES[mode]
    g = _gen(22 + H)
    B, E = 2, 32 * H
    for Pq in (1, 63, 64, 65, 127, 128, 129):
        for Pk in (1, 127, 128, 129, 300):
            q = _randn_tf32(g, B, Pq, E, scale=0.5).to(cuda)
            k, v = _randn_tf32(g, B, Pk, E).to(cuda), _randn_tf32(g, B, Pk, E).to(cuda)
            mask = torch.zeros(B, Pk, dtype=torch.uint8)
            mask[0] = (torch.rand(Pk, generator=g) < 1 / 3).to(torch.uint8)
            mask[0, 0] = 0
            _check_attention(q, k, v, mask.to(cuda), H, mode, 'attention H=%d Pq=%d Pk=%d' % (H, Pq, Pk))


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_attention_masks(cuda, mode):
    """rows with every key masked (NaN, as torch), valid keys only in the third 128-key block (the first two blocks leave the running
    max at -inf), only the last key valid"""
    mode = MODES[mode]
    g = _gen(23)
    B, Pq, Pk, H, E = 3, 77, 400, 8, 256
    q = _randn_tf32(g, B, Pq, E, scale=0.5).to(cuda)
    k, v = _randn_tf32(g, B, Pk, E).to(cuda), _randn_tf32(g, B, Pk, E).to(cuda)
    mask = torch.ones(B, Pk, dtype=torch.uint8)
    mask[1, 256:384] = 0
    mask[2, Pk - 1] = 0
    out = ops.attention(q, k, v, mask.to(cuda), H, mode=mode)
    assert bool(torch.isnan(out[0]).all()), 'every key masked: NaN like torch'
    _check_attention(q, k, v, mask.to(cuda), H, mode, 'attention masks')


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_attention_large_logits(cuda, mode):
    """logits up to |s| ~ 80, growing along the keys, so the running maximum moves block after block and the rescale exp(m_old - m_new)
    carries the earlier blocks; TF32-representable q / k / v keep the bound sharp"""
    mode = MODES[mode]
    g = _gen(24)
    B, Pq, Pk, H, E = 2, 130, 700, 8, 256

    def max_logit(q, k):
        return (q.view(B, Pq, H, 32).transpose(1, 2).double() @ k.view(B, Pk, H, 32).permute(0, 2, 3, 1).double()).abs().max().item()
    q = torch.randn(B, Pq, E, generator=g)
    k = torch.randn(B, Pk, E, generator=g) * torch.linspace(0.2, 1.0, Pk)[None, :, None]
    v = torch.randn(B, Pk, E, generator=g)
    q = q * (80.0 / max_logit(q, k))
    q, k, v = (ops.round_tf32(t) for t in (q, k, v))
    s_max = max_logit(q, k)
    assert 70 < s_max < 90, s_max
    _check_attention(q.to(cuda), k.to(cuda), v.to(cuda), None, H, mode, 'attention |s| <= %.0f' % s_max)


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_attention_unsupported_layouts(cuda, mode):
    """head_dim != 32 is refused in both modes; a row stride that is not a multiple of 4 floats is refused by the TF32 kernel (its TMA
    loads need 16-byte rows) and computed correctly by the fp32 one"""
    mode = MODES[mode]
    g = _gen(25)
    B, Pq, Pk = 2, 70, 150
    q, k, v = (torch.randn(B, P, 128, generator=g).to(cuda) for P in (Pq, Pk, Pk))
    with pytest.raises(RuntimeError, match='head_dim'):
        ops.attention(q, k, v, None, 8, mode=mode)               # dh = 16
    # q contiguous; k and v: the first 256 columns of rows of 257 floats
    q = (torch.randn(B, Pq, 256, generator=g) * 0.5).to(cuda)
    k, v = (torch.randn(B, Pk, 257, generator=g).to(cuda)[:, :, :256] for _ in range(2))
    if mode == TF32:
        with pytest.raises(RuntimeError, match='16-byte'):
            ops.attention(q, k, v, None, 8, mode=mode)
    else:
        _check_attention(q, k, v, None, 8, mode, 'attention fp32, k / v row stride 257')


# ---------------------------------------------------------------------------------------------------------------------------------
# LayerNorm(x + r)
# ---------------------------------------------------------------------------------------------------------------------------------
def _layernorm_ref(x, r, gamma, beta, eps):
    """float64 LayerNorm(x + r) and its bound.  The kernel (one warp per row, C / 32 values per lane) rounds t = x + r (u |t|), sums
    sequentially per lane then over a 5-level shuffle tree and divides: |dmean| <= (C/32 + 8) u mean|t| (incl. the rounding of t);
    d = t - mean: E_d = u max|t| + |dmean| + u max|d|.  var: FMA chains + tree + division, (C/32 + 7) u var, plus 2 E_d mean|d| + E_d^2
    from the error in d.  rstd = rsqrtf(var + eps) (2 ulp) after a rounded add: relative rho = dvar / (2 (var + eps)) + 6 u.
    y = (d * rstd) * gamma + beta, three roundings: |dy| <= |gamma| rstd (E_d + |d| rho) + 3 u (|d rstd gamma| + |beta|).
    Doubled for the second-order terms dropped above."""
    C = x.shape[1]
    t = x.to(F64) + (r.to(F64) if r is not None else 0)
    mean = t.mean(dim=1, keepdim=True)
    d = t - mean
    var = (d * d).mean(dim=1, keepdim=True)
    rstd = (var + eps).rsqrt()
    y = d * rstd * gamma.to(F64) + beta.to(F64)
    dmean = (C / 32 + 8) * U * t.abs().mean(dim=1, keepdim=True)
    e_d = U * t.abs().amax(dim=1, keepdim=True) + dmean + U * d.abs().amax(dim=1, keepdim=True)
    dvar = (C / 32 + 7) * U * var + 2 * e_d * d.abs().mean(dim=1, keepdim=True) + e_d * e_d
    rho = dvar / (2 * (var + eps)) + 6 * U
    bound = gamma.to(F64).abs() * rstd * (e_d + d.abs() * rho) + 3 * U * ((d * rstd * gamma.to(F64)).abs() + beta.to(F64).abs())
    return y, 2 * bound


@pytest.mark.parametrize('C', [32, 100, 256, 512])
def test_layernorm_residual(cuda, C):
    """C = 512 (the kernel's register limit), C % 32 != 0, r = None, and rows of mean 1e3 / variance 1e-2 (a one-pass variance
    E[t^2] - mean^2 would lose it entirely)"""
    g = _gen(31 + C)
    M = 300
    x, r = torch.randn(M, C, generator=g), torch.randn(M, C, generator=g)
    x[:50] = 1e3 + 0.1 * torch.randn(50, C, generator=g)
    r[:50] *= 1e-3
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    x, r, gamma, beta = x.to(cuda), r.to(cuda), gamma.to(cuda), beta.to(cuda)
    for rr in (r, None):
        y = ops.layernorm_residual(x, rr, gamma, beta, 1e-5)
        ref, bound = _layernorm_ref(x, rr, gamma, beta, 1e-5)
        _assert_within(y, ref, bound, 'layernorm C=%d r=%s' % (C, 'None' if rr is None else 'given'))

"""CPU checks of the dense-conv test arithmetic (the conv2d section of tests/spconv_arith.py), so that the element-wise GPU checks of
the dense convolutions (tests/test_gpu_conv2d_kernels.py and the conv tests of test_gpu_det.py, test_gpu_conv_halo_n256.py,
test_gpu_conv_epilogue.py) cannot pass vacuously:

- the exact operands in dense layout are exact up to cin = 512 with 9 taps, and their contract sums give the same float32 bits in
  any order and with truncating adds;
- the fp32 and tf32 bounds accept a float32 emulation of the kernels' arithmetic (a sequential FMA chain; 8-product MMA steps
  added into a truncating fp32 accumulator), with ReLU on and off, TF32-exact and raw inputs, both forms of the fp32 epilogue;
- the bounds reject an emulation that drops one tap, reads the weights without RN to TF32, RNA-rounds an output without ReLU, or
  truncates a ReLU output instead of RNA-rounding it."""
import pytest
import torch

from tests import spconv_arith as sa
from tests.util import assert_within

F64 = torch.float64


def _out_hw(H, W, k, stride, pad):
    return (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1


def _emulate(mode, x, w, stride, pad, scale, shift, relu, drop_tap=None, weight_read='rn', out_round='contract', fma=False,
             order='forward'):
    """float32 emulation of a dense conv (x (B, H, W, cin), w (cout, cin, KH, KW)) over the (tap, channel) reduction in the kernels'
    order: fp32 one FMA per product; tf32 the tensor core's reads T(x), RN(w) (weight_read='trunc': T(w)), then one truncating add of
    each 8-product MMA step.  Then * scale, + shift in fp32 (fma: one rounding), ReLU and the output rounding ('contract':
    sa.output_bits; 'rna', 'trunc': that rounding to TF32 whatever relu is)"""
    B, H, W, cin = x.shape
    cout, _, KH, KW = w.shape
    K = KH * KW
    Ho, Wo = _out_hw(H, W, KH, stride, pad)
    if mode == 'fp32':
        xa, wb = x, w
    else:
        xa, wb = sa.trunc_tf32(x), (sa.rn_tf32(w) if weight_read == 'rn' else sa.trunc_tf32(w))
    cols = torch.nn.functional.unfold(xa.to(F64).permute(0, 3, 1, 2), (KH, KW), padding=pad, stride=stride)   # (B, cin K, L)
    cols = cols.view(B, cin, K, -1).permute(0, 3, 2, 1).reshape(-1, K, cin).clone()                         # (B L, K, cin)
    if drop_tap is not None:
        cols[:, drop_tap] = 0
    cols = cols.reshape(-1, K * cin)
    wk = wb.to(F64).reshape(cout, cin, K).permute(2, 1, 0).reshape(K * cin, cout)
    idx = list(range(K * cin)) if mode == 'fp32' else list(range(0, K * cin, 8))
    if order == 'reverse':
        idx = idx[::-1]
    acc = torch.zeros(cols.shape[0], cout, dtype=torch.float32)
    for i in idx:
        if mode == 'fp32':
            acc = (acc.to(F64) + cols[:, i:i + 1] * wk[i:i + 1]).float()
        else:
            acc = sa.trunc32(acc.to(F64) + cols[:, i:i + 8] @ wk[i:i + 8])
    if fma:
        o = (acc.to(F64) * scale.to(F64) + shift.to(F64)).float()
    else:
        o = acc * scale + shift
    if relu:
        o = o.clamp_min(0)
    if out_round == 'contract':
        o = sa.output_bits(mode, o, relu)
    elif out_round == 'rna':
        o = sa.rna_tf32(o)
    elif out_round == 'trunc':
        o = sa.trunc_tf32(o)
    return o.view(B, Ho, Wo, cout)


def _check(mode, got, x, w, stride, pad, scale, shift, relu, what):
    return sa.assert_conv2d(got, x, w, stride, pad, scale, shift, relu, mode, what)


def _problem(g, cin=16, cout=8, H=7, W=6, B=2, x_exact=True):
    x = torch.randn(B, H, W, cin, generator=g) * torch.logspace(-2, 2, B * H * W).view(B, H, W, 1)
    if x_exact:
        x = sa.rn_tf32(x)                                   # a ReLU output of the previous TF32 conv
    w = torch.randn(cout, cin, 3, 3, generator=g) / (9 * cin) ** 0.5
    return x, w, torch.randn(cout, generator=g), torch.randn(cout, generator=g)


# ---- exactness of the exact operands at dense shapes -------------------------------------------------------------------------
@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
@pytest.mark.parametrize('cin,k,stride,pad', [(512, 3, 1, 1), (32, 3, 2, 1), (64, 3, 1, 0), (128, 1, 1, 0)])
def test_exact_dense_operands_sum_in_any_order(mode, cin, k, stride, pad):
    g = torch.Generator().manual_seed(cin + 10 * k + stride)
    B, H, W, cout = 2, 5, 7, 8
    x, w, scale, shift = sa.exact_dense(g, mode, B, H, W, cin, cout, k, k)
    amax = sa.assert_exact_dense(mode, x, w, stride, pad)
    assert amax > 2.0 ** 7 if cin == 512 else amax > 0                     # the budget is used, not just met
    y, _ = sa.dense_contract64(mode, x, w, stride, pad)
    for relu in (False, True):
        o = sa.epilogue_exact(mode, y, scale, shift, None, relu)
        assert torch.equal(o, o.float().to(F64)), 'the epilogue must be exact'
        want = sa.output_bits(mode, o.float(), relu)
        if mode == 'tf32' and relu:
            assert (want != o.float()).float().mean() > 0.2, 'the output rounding must be exercised'
        if cin <= 128:
            for order in ('forward', 'reverse'):
                got = _emulate(mode, x, w, stride, pad, scale, shift, relu, order=order)
                assert torch.equal(got, want), order


def test_exact_dense_deconv_operands():
    g = torch.Generator().manual_seed(5)
    for mode in ('fp32', 'tf32'):
        x, w, scale, shift = sa.exact_dense(g, mode, 2, 3, 5, 256, 12, 2, 2, transposed=True)
        assert w.shape == (256, 12, 2, 2)
        sa.assert_exact_dense(mode, x, w, transposed=True)
        y, _ = sa.dense_contract64(mode, x, w, transposed=True)
        assert y.shape == (2, 6, 10, 12) and torch.equal(y, y.float().to(F64))


# ---- the bounds accept the kernels' arithmetic ---------------------------------------------------------------------------------
@pytest.mark.parametrize('stride,pad', [(1, 1), (2, 1), (1, 0)])
@pytest.mark.parametrize('mode,x_exact', [('fp32', False), ('tf32', True), ('tf32', False)])
def test_bound_accepts_emulation(mode, x_exact, stride, pad):
    g = torch.Generator().manual_seed(3 * stride + pad + 7 * x_exact)
    for relu in (False, True):
        for fma in ((False, True) if mode == 'fp32' else (False,)):
            x, w, scale, shift = _problem(g, x_exact=x_exact)
            got = _emulate(mode, x, w, stride, pad, scale, shift, relu, fma=fma)
            worst = _check(mode, got, x, w, stride, pad, scale, shift, relu, '%s relu=%d fma=%d' % (mode, relu, fma))
            assert worst > 0


# ---- the bounds reject the defects they are meant to find -----------------------------------------------------------------------
def _positive(g, cin=16, cout=8, H=7, W=6, B=2):
    """one-sign operands: TF32-exact inputs and weights, positive scale, no shift"""
    x = sa.rn_tf32(torch.rand(B, H, W, cin, generator=g) + 0.5)
    w = sa.rn_tf32((torch.rand(cout, cin, 3, 3, generator=g) + 0.5) / (9 * cin) ** 0.5)
    return x, w, torch.rand(cout, generator=g) + 0.5, torch.zeros(cout)


@pytest.mark.parametrize('mode', ['fp32', 'tf32'])
def test_bound_rejects_a_dropped_tap(mode):
    g = torch.Generator().manual_seed(21)
    x, w, scale, shift = _positive(g)
    for tap in (0, 4, 8):
        got = _emulate(mode, x, w, 1, 1, scale, shift, False, drop_tap=tap)
        with pytest.raises(AssertionError, match='largest err/bound'):
            _check(mode, got, x, w, 1, 1, scale, shift, False, 'tap %d dropped' % tap)


def test_bound_rejects_unrounded_weights():
    """weights with a mantissa in [1, 1.1) and 0.75 to 0.95 TF32 ulp above the TF32 grid: the truncating read of the unrounded weight
    errs by more than 2^-11 of it, RN by less than 2^-12"""
    g = torch.Generator().manual_seed(22)
    x, _, scale, shift = _positive(g)
    t = sa.rn_tf32((1 + 0.1 * torch.rand(8, 16, 3, 3, generator=g)) * 2.0 ** torch.randint(-5, -2, (8, 16, 3, 3), generator=g))
    ulp = torch.ldexp(torch.ones_like(t), torch.frexp(t).exponent - 11)
    w = (t + ulp * (0.75 + 0.2 * torch.rand(t.shape, generator=g))).float()
    _check('tf32', _emulate('tf32', x, w, 1, 1, scale, shift, False), x, w, 1, 1, scale, shift, False, 'RN weights')
    got = _emulate('tf32', x, w, 1, 1, scale, shift, False, weight_read='trunc')
    with pytest.raises(AssertionError, match='largest err/bound'):
        _check('tf32', got, x, w, 1, 1, scale, shift, False, 'truncated weights')


def _shift_dominated(g, lo, width, cin=16, cout=8, H=7, W=6, B=2):
    """small TF32-exact inputs and a full-precision shift in [lo, lo + width): the output is mostly the shift, so its rounding is not
    hidden under the operand term of the bound (the CenterHead's last conv: heatmap bias -2.19, small conv contributions)"""
    x = sa.rn_tf32(torch.randn(B, H, W, cin, generator=g) * 1e-3)
    w = torch.randn(cout, cin, 3, 3, generator=g) / (9 * cin) ** 0.5
    return x, w, torch.ones(cout), lo + width * torch.rand(cout, generator=g)


def test_bound_rejects_a_rounded_output_without_relu():
    g = torch.Generator().manual_seed(23)
    x, w, scale, shift = _shift_dominated(g, 1.0, 1.0)
    _check('tf32', _emulate('tf32', x, w, 1, 1, scale, shift, False), x, w, 1, 1, scale, shift, False, 'stored unrounded')
    got = _emulate('tf32', x, w, 1, 1, scale, shift, False, out_round='rna')
    with pytest.raises(AssertionError, match='largest err/bound'):
        _check('tf32', got, x, w, 1, 1, scale, shift, False, 'RNA without ReLU')


def test_bound_rejects_a_truncated_relu_output():
    g = torch.Generator().manual_seed(24)
    x, w, scale, shift = _shift_dominated(g, 1.0, 0.25)
    _check('tf32', _emulate('tf32', x, w, 1, 1, scale, shift, True), x, w, 1, 1, scale, shift, True, 'RNA with ReLU')
    got = _emulate('tf32', x, w, 1, 1, scale, shift, True, out_round='trunc')
    with pytest.raises(AssertionError, match='largest err/bound'):
        _check('tf32', got, x, w, 1, 1, scale, shift, True, 'truncated ReLU output')

"""CPU checks of the sparse-conv test arithmetic (tests/spconv_arith.py), so that the GPU tests that rely on it cannot pass
vacuously:

- the exact-operand generators really are exact: every contract product is exact in fp32, and the contract sum in float32 gives
  the same bits in forward order, in reverse order, pairwise and with truncating adds;
- each mode's bound accepts a float32 emulation of that mode's arithmetic with truncating accumulation per MMA step;
- each bound rejects an emulation that drops one contract term (or, for the one-term modes, one reduction step), on operands
  whose dropped terms all share one sign."""
import pytest
import torch

from tests import spconv_arith as sa
from tests.util import assert_within

F64 = torch.float64


def _table(g, K, n_out, n_in, p=0.6):
    """k-major (K, n_out) neighbour table with random pairs (each offset maps an output to at most one input)"""
    j = torch.randint(0, n_in, (K, n_out), generator=g, dtype=torch.int32)
    return torch.where(torch.rand(K, n_out, generator=g) < p, j, torch.full_like(j, -1))


def _products(mode, nbr, x, w, x_is_planes=False):
    """(n_out, cout, L) float64 products of the contract, zero where a pair is missing"""
    K, n_out = nbr.shape
    cols = []
    for a, b in sa.pieces(mode, x, w, x_is_planes):
        for k in range(K):
            j = nbr[k].long()
            ga = torch.where((j >= 0)[:, None], a[j.clamp_min(0)], torch.zeros(()))        # (n_out, cin)
            cols.append(ga.to(F64)[:, None, :] * b[k].to(F64).t()[None, :, :])           # (n_out, cout, cin)
    return torch.cat(cols, 2)


def _sum32(p, order, trunc=False):
    if order == 'pairwise':
        t = p.float()
        while t.shape[-1] > 1:
            if t.shape[-1] % 2:
                t = torch.cat([t, torch.zeros_like(t[..., :1])], -1)
            t = (t[..., 0::2].to(F64) + t[..., 1::2].to(F64)).float()
        return t[..., 0]
    idx = range(p.shape[-1]) if order == 'forward' else reversed(range(p.shape[-1]))
    acc = torch.zeros(p.shape[:-1], dtype=torch.float32)
    for i in idx:
        s = acc.to(F64) + p[..., i]
        acc = sa.trunc32(s) if trunc else s.float()
    return acc


@pytest.mark.parametrize('mode', sa.MODES)
@pytest.mark.parametrize('K,cin', [(27, 128), (27, 5), (3, 128)])
def test_exact_operands_sum_in_any_order(mode, K, cin):
    g = torch.Generator().manual_seed(K * 1000 + cin)
    n_in, n_out, cout = 40, 24, 16
    x, w, scale, shift, res = sa.exact_operands(g, mode, n_in, cin, cout, K, n_out)
    nbr = _table(g, K, n_out, n_in, p=0.9)
    nbr[:, 0] = torch.randint(0, n_in, (K,), generator=g, dtype=torch.int32)     # one output with every offset live
    p = _products(mode, nbr, x, w)
    assert torch.equal(p, p.float().to(F64)), 'a contract product is not exact in fp32'
    exact = p.sum(-1)
    assert torch.equal(exact, exact.float().to(F64))
    for order, trunc in (('forward', False), ('reverse', False), ('pairwise', False), ('forward', True), ('reverse', True)):
        assert torch.equal(_sum32(p, order, trunc).to(F64), exact), (order, trunc)
    assert torch.equal(exact, sa.contract64(mode, nbr, x, w))
    # the epilogue is exact too, and x . w differs from the contract where the mode drops terms
    o = sa.epilogue_exact(mode, exact, scale, shift, res, True)
    assert torch.equal(o, o.float().to(F64))
    if sa.dropped(mode, x, w):
        assert not torch.equal(sa.conv64(nbr, x, w), exact), 'the dropped terms must be non-zero'
    if mode in ('tf32', 'bf16'):
        stored = sa.output_bits(mode, o.float()).float()
        assert (stored != o.float()).float().mean() > 0.2, 'the output rounding must be exercised'
    assert (p.abs().sum(-1) < 2.0 ** 9).all()


# ---- float32 emulation of each mode's arithmetic ------------------------------------------------------------------------------
def _emulate(mode, nbr, x, w, scale, shift, res, relu, x_is_planes=False, drop_piece=None, drop_last_step=False):
    """the mode's arithmetic in float32: fp32 a sequential FMA chain over (k, c); the tensor-core modes one truncating fp32 add of
    each MMA step's (exact) chunk sum, the chunks running over the concatenated (offset, padded channel) dimension; then the
    epilogue with round-to-nearest float32 operations and the output rounding"""
    K, n_out = nbr.shape
    cin = w.shape[1]
    cin_pad = 8 if cin <= 8 else cin
    ps = sa.pieces(mode, x, w, x_is_planes)
    if drop_piece is not None:
        ps = [pq for i, pq in enumerate(ps) if i != drop_piece]
    gathered = []
    for a, b in ps:
        ga = torch.zeros(n_out, K, cin_pad, dtype=F64)
        wb = torch.zeros(K, cin_pad, w.shape[2], dtype=F64)
        for k in range(K):
            j = nbr[k].long()
            ok = j >= 0
            ga[ok, k, :cin] = a[j[ok]].to(F64)
        wb[:, :cin] = b.to(F64)
        gathered.append((ga.reshape(n_out, -1), wb.reshape(K * cin_pad, -1)))
    acc = torch.zeros(n_out, w.shape[2], dtype=torch.float32)
    L = K * cin_pad
    if mode == 'fp32':
        (ga, wb), = gathered
        last = L - (cin_pad - cin) - 1
        for i in range(L):
            if drop_last_step and i == last:
                continue
            acc = (acc.to(F64) + ga[:, i:i + 1] * wb[i:i + 1]).float()          # FMA: one rounding
    else:
        ch = 8 if mode in ('tf32', 'tf32x3') else 16
        steps = list(range(0, L, ch))
        if drop_last_step:
            steps = steps[:-1]
        for s in steps:
            for ga, wb in gathered:
                acc = sa.trunc32(acc.to(F64) + ga[:, s:s + ch] @ wb[s:s + ch])
    if mode in sa.PLANES:
        o = (acc.to(F64) * scale.to(F64) + shift.to(F64)).float()                # fma
    else:
        o = acc * scale + shift
    for r in sa.residual_pieces(mode, res):
        o = o + r
    if relu:
        o = o.clamp_min(0)
    return sa.stored_value(mode, sa.output_bits(mode, o), w.shape[2])


def _problem(g, mode, K, cin, n_in=60, n_out=50, cout=16, one_sign=False):
    if one_sign:
        # x = t + delta, delta in (0.25, 0.45) ulp of t in the mode's operand format: every low piece of x (A_lo, p1) is positive,
        # as is every weight piece; then every dropped term has one sign
        bits = 7 if mode in sa.PLANES else 10

        def above(t):
            t = t.float()
            t = t.to(torch.bfloat16).float() if mode in sa.PLANES else sa.rn_tf32(t)
            ulp = torch.ldexp(torch.ones_like(t), torch.frexp(t).exponent - 1 - bits)
            return t + ulp * (0.25 + 0.2 * torch.rand(t.shape, generator=g))
        x = above(torch.rand(n_in, cin, generator=g) + 0.5)
        w = above((torch.rand(K, cin, cout, generator=g) + 0.5) / (K * cin) ** 0.5)
        scale, shift = torch.rand(cout, generator=g) + 0.5, torch.rand(cout, generator=g)
        res = None
    else:
        x = torch.randn(n_in, cin, generator=g) * torch.logspace(-2, 2, n_in)[:, None]
        w = torch.randn(K, cin, cout, generator=g) / (K * cin) ** 0.5
        scale, shift = torch.randn(cout, generator=g), torch.randn(cout, generator=g)
        res = torch.randn(n_out, cout, generator=g)
    if mode == 'tf32':
        x = sa.rn_tf32(x)                # what every TF32 layer of the backbone reads
    nbr = _table(g, K, n_out, n_in)
    return x.float(), w.float(), scale.float(), shift.float(), res, nbr


def _reference(mode, nbr, x, w, scale, shift, res, relu):
    """float64 x . w epilogue, with x the layer's stored input (bf16 modes: the planes) and the residual as stored"""
    xr = x
    if mode in sa.PLANES:
        p0, p1 = sa.split_bf16(x)
        planes = torch.stack([p0, p1] if mode == 'bf16x2' else [p0], 1)
        xr = planes.to(F64).sum(1)
    y = sa.conv64(nbr, xr, w)
    A = sa.conv64(nbr, xr.abs(), w.abs())
    r = None
    if res is not None:
        r = sum(p.to(F64) for p in sa.residual_pieces(mode, res))
    o = y * scale.to(F64) + shift.to(F64) + (0 if r is None else r)
    if relu:
        o = o.clamp_min(0)
    x_in = planes if mode in sa.PLANES else x
    return o, A, (None if r is None else r.abs()), x_in


@pytest.mark.parametrize('mode', sa.MODES)
@pytest.mark.parametrize('K,cin', [(27, 16), (27, 5), (3, 32)])
def test_bound_accepts_emulation(mode, K, cin):
    g = torch.Generator().manual_seed(7 * K + cin)
    for relu in (False, True):
        x, w, scale, shift, res, nbr = _problem(g, mode, K, cin)
        ref, A, r_abs, x_in = _reference(mode, nbr, x, w, scale, shift, res, relu)
        got = _emulate(mode, nbr, x_in, w, scale, shift, res, relu, x_is_planes=mode in sa.PLANES)
        b = sa.bound(mode, K, cin, A, scale, shift, r_abs, got.abs())
        worst = assert_within(got, ref, b, '%s K=%d cin=%d relu=%d' % (mode, K, cin, relu))
        assert worst > 0 or mode == 'fp32'


@pytest.mark.parametrize('mode', sa.MODES)
@pytest.mark.parametrize('K,cin', [(27, 16), (3, 32)])
def test_bound_rejects_a_dropped_term(mode, K, cin):
    g = torch.Generator().manual_seed(11 * K + cin)
    x, w, scale, shift, res, nbr = _problem(g, mode, K, cin, one_sign=True)
    ref, A, r_abs, x_in = _reference(mode, nbr, x, w, scale, shift, res, False)
    n_pieces = len(sa.pieces(mode, x, w))
    variants = [dict(drop_piece=i) for i in range(n_pieces)] if n_pieces > 1 else [dict(drop_last_step=True)]
    for kw in variants:
        got = _emulate(mode, nbr, x_in, w, scale, shift, res, False, x_is_planes=mode in sa.PLANES, **kw)
        b = sa.bound(mode, K, cin, A, scale, shift, r_abs, got.abs())
        with pytest.raises(AssertionError, match='largest err/bound'):
            assert_within(got, ref, b, '%s %s' % (mode, kw))


@pytest.mark.parametrize('mode', ['tf32x3', 'bf16x2'])
def test_fp32_level_bounds_are_below_the_single_pass_operand_term(mode):
    """at every production shape the fp32-level modes' whole pre-epilogue bound stays below the single-pass operand error, so the
    element-wise checks can tell tf32x3 from tf32 and bf16x2 from bf16"""
    for K, cin in ((27, 5), (27, 16), (27, 32), (27, 64), (27, 128), (3, 128)):
        c = sa.operand_coef(mode) + sa.accumulation_coef(mode, K, cin)
        assert c < sa.single_pass_coef(mode), (mode, K, cin, c)

"""The arithmetic contract of the sparse-conv forward kernels, per compute mode, and the element-wise error bounds derived from it.

Every mode computes out[o] = epilogue(sum_k sum_c x[nbr[k][o], c] W[k, c, :]) from operand pieces:
    fp32     x . w                                  exact-fp32 FMA (csrc/spconv.cu)
    tf32     T(x) . RN(w)                           one TF32 pass; T = the tensor core's truncating read, RN = pack_spconv_weight
    tf32x3   A_lo W_hi + A_hi W_lo + A_hi W_hi      A_hi = RNA(x), A_lo = RNA(x - A_hi), W split by RN; A_lo W_lo is dropped
    bf16x2   p0 w0 + p0 w1 + p1 w0                  the input planes as stored, W split by RN_bf16; p1 w1 is dropped
    bf16     p0 w0
then out = relu(y * scale + shift + residual) (bf16 modes: one fma, then plane 0 and plane 1 of the residual), rounded to the
output format: RNA_tf32 for tf32, planes p0 = RN_bf16(o), p1 = RN_bf16(o - p0) for bf16x2, RN_bf16 for bf16.

The helpers here run on CPU or GPU tensors alike.  u = 2^-24 is the fp32 unit roundoff."""
import torch

from detzero_b200 import ops

F64 = torch.float64
U = 2.0 ** -24
MODES = ('fp32', 'tf32', 'tf32x3', 'bf16x2', 'bf16')
PLANES = {'bf16x2': 2, 'bf16': 1}
#: safety factor on the tensor core's accumulation: every serial MMA step (one wgmma k-chunk of 8 TF32 / 16 bf16 products added
#: into the fp32 accumulator) may err by TC_SAFETY u times the sum of the magnitudes it has accumulated, <= TC_SAFETY u A
TC_SAFETY = 4


# ---- roundings ---------------------------------------------------------------------------------------------------------------
def rn_tf32(t):
    """round to nearest, ties to even, to TF32 (ops.round_tf32, what pack_spconv_weight and dz_round_tf32 do)"""
    return ops.round_tf32(t.float())


def rna_tf32(t):
    """round to nearest, ties away from zero, to TF32 (cvt.rna.tf32.f32) of finite values"""
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def trunc_tf32(t):
    """the tensor core's read of an fp32 operand: the low 13 mantissa bits dropped"""
    return (t.float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def trunc32(v64):
    """float64 -> float32 rounded toward zero (a truncating fp32 add)"""
    f = v64.float()
    over = f.to(F64).abs() > v64.abs()
    return torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)


def split_bf16(t):
    """(p0, p1) = (RN_bf16(t), RN_bf16(t - p0)) as float32 (ops.to_planes, pack_spconv_weight)"""
    t = t.float()
    p0 = t.to(torch.bfloat16).float()
    return p0, (t - p0).to(torch.bfloat16).float()


# ---- contract -----------------------------------------------------------------------------------------------------------------
def pieces(mode, x, w, x_is_planes=False):
    """the contract's (input piece, weight piece) pairs, float32.  x (n, cin) is the layer's fp32 input -- or, for the bf16 modes
    with x_is_planes, a (n, P, cin) stack of the stored planes; w (K, cin, cout) fp32"""
    if mode == 'fp32':
        return [(x, w)]
    if mode == 'tf32':
        return [(trunc_tf32(x), rn_tf32(w))]
    if mode == 'tf32x3':
        ah = rna_tf32(x)
        al = rna_tf32(x - ah)
        wh = rn_tf32(w)
        return [(al, wh), (ah, rn_tf32(w - wh)), (ah, wh)]
    if x_is_planes:
        p0, p1 = x[:, 0], (x[:, 1] if x.shape[1] > 1 else torch.zeros_like(x[:, 0]))
    else:
        p0, p1 = split_bf16(x)
    w0, w1 = split_bf16(w)
    if mode == 'bf16x2':
        return [(p0, w0), (p0, w1), (p1, w0)]
    assert mode == 'bf16', mode
    return [(p0, w0)]


def dropped(mode, x, w):
    """the (input piece, weight piece) pairs x . w has and the contract drops (non-empty for tf32x3, bf16x2, bf16)"""
    if mode == 'tf32x3':
        ah = rna_tf32(x)
        wh = rn_tf32(w)
        return [(rna_tf32(x - ah), rn_tf32(w - wh))]
    if mode in PLANES:
        p0, p1 = split_bf16(x)
        w0, w1 = split_bf16(w)
        return [(p1, w1)] if mode == 'bf16x2' else [(p0, w1), (p1, w0), (p1, w1)]
    return []


def conv64(nbr, x, w):
    """float64 sum_k x[nbr[k][o]] @ w[k] over the k-major table nbr (K, n_out), -1 = no neighbour"""
    K, n_out = nbr.shape
    y = torch.zeros(n_out, w.shape[2], dtype=F64, device=x.device)
    x64, w64 = x.to(F64), w.to(F64)
    for k in range(K):
        j = nbr[k].long()
        ok = j >= 0
        if bool(ok.any()):
            y[ok] += x64[j[ok]] @ w64[k]
    return y


def contract64(mode, nbr, x, w, x_is_planes=False):
    y = None
    for a, b in pieces(mode, x, w, x_is_planes):
        t = conv64(nbr, a, b)
        y = t if y is None else y + t
    return y


def residual_pieces(mode, r):
    """the residual as the epilogue adds it: one fp32 value, or plane 0 then plane 1 (bf16x2) / plane 0 (bf16)"""
    if r is None:
        return []
    if mode in PLANES:
        p0, p1 = split_bf16(r)
        return [p0, p1] if mode == 'bf16x2' else [p0]
    return [r.float()]


def epilogue_exact(mode, y64, scale, shift, res, relu):
    """float64 epilogue for operands on which every step is exact (checked: the caller's result must be float32-representable)"""
    o = y64 * scale.to(F64) + shift.to(F64)
    for p in residual_pieces(mode, res):
        o = o + p.to(F64)
    if relu:
        o = o.clamp_min(0)
    return o


def output_bits(mode, o32, relu=True):
    """what the kernel stores for the fp32 epilogue value o32: float32 (rows, cout) or bf16 planes (rows, P * cout).  The sparse
    convs round every tf32 output; the dense tf32 convs round only a ReLU output (it feeds another TF32 conv), so relu=False
    stores the fp32 value as it is"""
    if mode == 'tf32':
        return rna_tf32(o32) if relu else o32
    if mode in PLANES:
        p0, p1 = split_bf16(o32)
        return (torch.cat([p0, p1], 1) if mode == 'bf16x2' else p0).to(torch.bfloat16)
    return o32


def stored_value(mode, out, cout):
    """float64 value of a stored output (planes summed)"""
    if mode in PLANES:
        P = PLANES[mode]
        o = out.to(F64).view(out.shape[0], P, cout)
        return o.sum(1)
    return out.to(F64)


# ---- exact operands -----------------------------------------------------------------------------------------------------------
#: exponent of the low piece of the split values: below half an ulp of a value in [1, 2) of the mode's operand format
LO = {'fp32': -12, 'tf32': -12, 'tf32x3': -12, 'bf16x2': -9, 'bf16': -9}


def exact_operands(g, mode, n_in, cin, cout, K, n_out):
    """x (n_in, cin), w (K, cin, cout), scale, shift (cout), residual (n_out, cout), all float32, such that every product of the
    contract is exact in fp32 and every partial sum stays below 2^23 units of its finest bit (so any order and any truncation of
    the additions is exact), the epilogue is exact (scale a power of two, shift and residual on the sum's grid) -- and the terms
    the contract drops are non-zero, so that x . w differs from the contract.

    Channel 0 carries the split values: x = a + c 2^LO with a in +-{1.25, 1.5, 1.75}, c = +-1 (tf32: c 2^-10, its inputs are
    TF32-representable; bf16: a +- 2^-7, so that plane 0 has its last bit); w = d + e 2^LO, d in +-{1.25, 1.5}, e = +-1 (fp32:
    plain d, and the split weights sit in channel 1, so the exact sum needs no bit below 2^(LO-2)).  Every other value is 0 or
    +-0.25.  The finest bit of any contract product is 2^(LO-2) (a, d have two fraction bits), and
    sum |terms| <= 27 (127 / 16 + 2.7) < 2^9 = 2^23 units of 2^-14 (tf32x3 at cin 128, the tightest case).  The epilogue keeps
    below 2^24 units: |y scale| <= 2^10 on a grid of 2^(LO-2) |scale|.  The sums of tf32 and bf16 need more bits than their
    output format holds, so the output rounding is exercised."""
    def pm(shape, vals):
        v = torch.tensor(vals, dtype=torch.float32)
        return v[torch.randint(0, len(vals), shape, generator=g)] * (torch.randint(0, 2, shape, generator=g) * 2 - 1).float()
    lo = 2.0 ** LO[mode]
    x = pm((n_in, cin), [0.0, 0.25, 0.25])
    w = pm((K, cin, cout), [0.0, 0.25, 0.25])
    xa = pm((n_in,), [1.25, 1.5, 1.75])
    xc = pm((n_in,), [1.0]) * lo
    wd = pm((K, cout), [1.25, 1.5])
    we = pm((K, cout), [1.0]) * lo
    if mode == 'tf32':                  # TF32-representable, with its last bit: sums need more than 11 bits, RNA is exercised
        xc = pm((n_in,), [1.0]) * 2.0 ** -10
    if mode == 'bf16':                  # a plane 0 with its last bit set, for the same reason: the sums need more than 8 bits
        xa = xa + pm((n_in,), [1.0]) * 2.0 ** -7
    x[:, 0] = xa + xc
    w[:, 0] = wd if mode == 'fp32' else wd + we
    if mode == 'fp32' and cin > 1:
        w[:, 1] = pm((K, cout), [1.25, 1.5]) + we
    scale = torch.tensor([0.5, 1.0, 2.0, -0.5, -1.0, -2.0])[torch.randint(0, 6, (cout,), generator=g)]
    shift = torch.randint(-16, 17, (cout,), generator=g).float() / 16
    if mode in PLANES:      # residual with a non-zero plane 1 (bf16x2): b + f 2^-9
        residual = pm((n_out, cout), [1.25, 1.5]) + pm((n_out, cout), [1.0]) * 2.0 ** -9
    else:
        residual = torch.randint(-32, 33, (n_out, cout), generator=g).float() / 16
    return x, w, scale, shift, residual


# ---- element-wise bounds ------------------------------------------------------------------------------------------------------
def mma_steps(mode, K, cin_pad):
    """serial MMA steps per output element: 4 wgmma k-chunks per 32-float (TF32) / 64-element (bf16) reduction block, 3 MMAs per
    chunk in the split modes"""
    if mode in ('tf32', 'tf32x3'):
        steps = 4 * -(-(K * cin_pad) // 32)
    else:
        steps = 4 * -(-(K * cin_pad) // 64)
    return steps * (3 if mode in ('tf32x3', 'bf16x2') else 1)


def accumulation_coef(mode, K, cin):
    """|computed sum - exact sum of the contract's products| <= coef * A, A = sum |x| |w|.
    fp32: K cin FMAs and K ceil(cin / 32) chunk adds, each rounding once (u); tensor-core modes: TC_SAFETY u per serial MMA step"""
    cin_pad = 8 if cin <= 8 else cin
    if mode == 'fp32':
        n = K * cin + K * -(-cin // 32)
        return n * U * (1 + n * U)
    return TC_SAFETY * mma_steps(mode, K, cin_pad) * U


def operand_coef(mode, x_tf32_exact=True):
    """|contract(x, w) - x . w| <= coef * A for the layer's input x as it is stored and its fp32 weights w.
    tf32: the weights RN to TF32 (2^-11), the input truncated unless TF32-representable (2^-10) and their product;
    tf32x3: |x - A_hi - A_lo| <= 2^-22 |x|, the same for W, and the dropped |A_lo W_lo| <= 2^-22 (1 + 2^-10) |x| |w|;
    bf16x2: the input is its two stored planes exactly, |w - w0 - w1| <= 2^-16 |w|, and the dropped
    |p1 w1| <= 2^-8 (1 + 2^-7) |x| * 2^-8 (1 + 2^-7) |w|;  bf16: |w - w0| <= 2^-8 |w|"""
    if mode == 'fp32':
        return 0.0
    if mode == 'tf32':
        ex = 0.0 if x_tf32_exact else 2.0 ** -10
        return ex + 2.0 ** -11 + ex * 2.0 ** -11
    if mode == 'tf32x3':
        return 2 * 2.0 ** -22 * (1 + 2.0 ** -21) + 2.0 ** -22 * (1 + 2.0 ** -10)
    if mode == 'bf16x2':
        return 2.0 ** -16 + 2.0 ** -16 * (1 + 2.0 ** -7) ** 2
    return 2.0 ** -8


def output_coef(mode, relu=True):
    """relative error of the output rounding: RNA to TF32 (2^-11; none for a dense conv without ReLU, see output_bits), two bf16
    planes (2^-16), one (2^-8)"""
    if mode == 'tf32' and not relu:
        return 0.0
    return {'fp32': 0.0, 'tf32x3': 0.0, 'tf32': 2.0 ** -11, 'bf16x2': 2.0 ** -16 * (1 + 2.0 ** -15), 'bf16': 2.0 ** -8}[mode]


def single_pass_coef(mode):
    """the operand term of the single-pass mode of the same family (RN-rounded input and weights): what an fp32-level mode's
    whole pre-epilogue bound must stay below, or the bound could not tell the two apart"""
    return {'tf32x3': 2.0 ** -11 + 2.0 ** -11, 'bf16x2': 2.0 ** -8}[mode]


def bound(mode, K, cin, A, scale, shift, res_abs, got_abs, x_tf32_exact=True, relu=True):
    """element-wise bound on |stored output - float64 x . w epilogue|.
    y = sum x w errs by (operand + accumulation) A; the epilogue multiplies that by |scale| and adds <= 3 roundings
    (u each) of |y scale|, + |shift|, + |residual|; ReLU is 1-Lipschitz; the output rounding adds output_coef |got|."""
    c = operand_coef(mode, x_tf32_exact) + accumulation_coef(mode, K, cin)
    sa = A * scale.abs().to(F64)
    b = c * sa + 3 * U * ((1 + c) * sa + shift.abs().to(F64) + (0 if res_abs is None else res_abs))
    return b + output_coef(mode, relu) * got_abs


# ---- dense conv2d / ConvTranspose2d (csrc/conv2d_tc.cu, csrc/bev.cu) ------------------------------------------------------------
# The dense convs follow the contract above with K = KH KW taps and no residual: tf32 is sum T(x) RN(w) (RN = pack_conv_weight /
# pack_deconv_weight) in 4 wgmma k-steps per 32-channel slice per tap, then __fmul_rn(., scale), __fadd_rn(., shift), fmaxf(., 0),
# and cvt.rna.tf32 only when ReLU is on; fp32 is one FMA chain over KH KW cin, then * scale, + shift (possibly contracted into
# one FMA: bound() allows three roundings) and ReLU, stored unrounded.  A ConvTranspose2d with kernel == stride has one tap per
# output (K = 1).  Tensors are NHWC: x (B, H, W, cin), outputs (B, Ho, Wo, cout); weights in torch layout, (cout, cin, KH, KW) or,
# transposed, (cin, cout, s, s).
def exact_dense(g, mode, B, H, W, cin, cout, KH, KW, transposed=False):
    """exact_operands in dense layout: x (B, H, W, cin), w (cout, cin, KH, KW) -- transposed: (cin, cout, KH, KW), KH = KW = s --,
    scale, shift (cout); tap k = r KW + s carries the split weight values of offset k"""
    x, w, scale, shift, _ = exact_operands(g, mode, B * H * W, cin, cout, KH * KW, 1)
    w = w.view(KH, KW, cin, cout)
    w = w.permute(2, 3, 0, 1) if transposed else w.permute(3, 2, 0, 1)
    return x.view(B, H, W, cin), w.contiguous(), scale, shift


def conv2d64(x, w, stride=1, pad=0, transposed=False):
    """float64 NHWC conv2d (or ConvTranspose2d with kernel == stride) of x and w, on their device"""
    x64, w64 = x.to(F64).permute(0, 3, 1, 2), w.to(F64)
    if transposed:
        y = torch.nn.functional.conv_transpose2d(x64, w64, stride=w.shape[2])
    else:
        y = torch.nn.functional.conv2d(x64, w64, stride=stride, padding=pad)
    return y.permute(0, 2, 3, 1)


def dense_contract64(mode, x, w, stride=1, pad=0, transposed=False):
    """(float64 contract sum, A = the sum of the magnitudes of its products) of a dense conv in mode fp32 / tf32"""
    y = A = None
    for a, b in pieces(mode, x, w):
        t = conv2d64(a, b, stride, pad, transposed)
        s = conv2d64(a.abs(), b.abs(), stride, pad, transposed)
        y, A = (t, s) if y is None else (y + t, A + s)
    return y, A


def _grid_bits(t, cdim):
    """per channel c (dimension cdim of t): (f, bits) with every t[c] an integer multiple of 2^-f and max |t[c]| 2^f < 2^bits"""
    t = t.to(F64).movedim(cdim, 0).reshape(t.shape[cdim], -1)
    f = torch.full((t.shape[0],), 99, dtype=torch.int64, device=t.device)
    for e in range(-30, 64):
        s = t * 2.0 ** e
        f[(s == s.round()).all(1) & (f == 99)] = e
    assert bool((f < 99).all())
    m = t.abs().amax(1) * torch.pow(2.0, f.to(F64))
    return f, torch.ceil(torch.log2(m + 1)).to(torch.int64)


def assert_exact_dense(mode, x, w, stride=1, pad=0, transposed=False):
    """the exactness budget of exact_operands at a dense shape, re-derived from the operands themselves rather than from the generator's
    argument: per input channel, the bits of the input piece plus the bits of the weight piece fit in 24 (every product is exact in
    fp32), and the largest sum of product magnitudes of an output stays below 2^24 units of the finest product bit (every partial
    sum in any order, rounded or truncated, is exact).  With the generator's values (channel 0: x in +-[1.25, 1.75] on 2^-10 (tf32)
    / 2^-12 (fp32), w in +-[1.25, 1.5] on 2^-2 after RN_tf32 (tf32) / channel 1 on 2^-12 (fp32); every other value 0 or +-0.25) an
    output sums at most K (1.76 * 1.5 + 0.25 * 1.51 + (cin - 2) / 16) < 9 * 35 = 315 at cin = 512, K = 9: below 2^9, on a grid of
    2^-12 (tf32) / 2^-14 (fp32), so below 2^21 / 2^23 units.  Returns the largest A"""
    wdim = 0 if transposed else 1
    f, A = None, None
    for a, b in pieces(mode, x, w):
        fa, ba = _grid_bits(a, a.dim() - 1)
        fb, bb = _grid_bits(b, wdim)
        assert int((ba + bb).max()) <= 24, 'a contract product is not exact in fp32'
        fab = int((fa + fb).max())
        f = fab if f is None else max(f, fab)
        s = conv2d64(a.abs(), b.abs(), stride, pad, transposed)
        A = s if A is None else A + s
    amax = float(A.max())
    assert amax * 2.0 ** f < 2.0 ** 24, ('partial sums may round', amax, f)
    return amax


def tf32_exact(t):
    """t is TF32-representable (the tensor core's truncating read of it is exact)"""
    return torch.equal(t, trunc_tf32(t))


def assert_conv2d(got, x, w, stride, pad, scale, shift, relu, mode, what, transposed=False):
    """element-wise check of a dense conv output got (B, Ho, Wo, cout) against the float64 conv of its input x as stored and its fp32
    weights w (torch layout), with bound(); x_tf32_exact is read off x itself.  One frame at a time on the device, so that the
    float64 operands of a 188 x 188 x 512 map stay small.  Returns the largest err / bound"""
    from tests.util import assert_within
    cout = got.shape[3]
    K = 1 if transposed else w.shape[2] * w.shape[3]
    cin = w.shape[0] if transposed else w.shape[1]
    dev = got.device
    one = torch.ones(cout, dtype=torch.float32, device=dev)
    scale = one if scale is None else scale.to(dev)
    shift = torch.zeros_like(one) if shift is None else shift.to(dev)
    exact = mode == 'tf32' and tf32_exact(x)
    w = w.to(dev)
    worst = 0.0
    for b in range(x.shape[0]):
        xb = x[b:b + 1].to(dev)
        y = conv2d64(xb, w, stride, pad, transposed)
        A = conv2d64(xb.abs(), w.abs(), stride, pad, transposed)
        ref = y * scale.to(F64) + shift.to(F64)
        if relu:
            ref = ref.clamp_min(0)
        gb = got[b:b + 1]
        bnd = bound(mode, K, cin, A, scale, shift, None, gb.to(F64).abs(), x_tf32_exact=exact, relu=relu)
        worst = max(worst, assert_within(gb, ref, bnd, '%s frame %d' % (what, b)))
    return worst

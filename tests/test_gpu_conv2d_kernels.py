"""Element-wise checks of every dense conv2d kernel -- k_conv2d_tf32<32|64|128, false|true>, k_conv2d_tf32_halo_n256<64|128> (TF32
wgmma, csrc/conv2d_tc.cu) and k_conv2d_f32<128,8 | 64,4 | 16,1> (exact fp32, csrc/bev.cu) -- against float64 restatements of the
same operation.

The arithmetic contract is that of the sparse convs (tests/spconv_arith.py) with K = KH KW taps and no residual:
    tf32   sum T(x) RN(w), T = the tensor core's truncating read, RN = pack_conv_weight / pack_deconv_weight; fp32 accumulation in
           4 wgmma k-steps per 32-channel slice per tap (mma_steps('tf32', KH KW, cin); a ConvTranspose2d with kernel == stride is
           one GEMM, K = 1); then __fmul_rn(acc, scale) (scale 1 when None), __fadd_rn(., shift), fmaxf(., 0), and cvt.rna.tf32
           ONLY when ReLU is on (the output feeds another TF32 conv); without ReLU the fp32 value is stored (the head's last conv).
    fp32   one FMA chain over KH KW cin, then * scale, + shift (the compiler may contract them into one FMA), ReLU, no rounding.
The input of the first BEV conv is not TF32-representable (bf16x2 sparse mode: plane 0 + plane 1); the contract there is the
truncating read, x_tf32_exact=False.  Every later conv reads an RNA-rounded ReLU output, which the production check asserts.

Two kinds of check:
- exact operands (spconv_arith.exact_dense): every contract product and partial sum is exact in fp32, so the stored bits are fixed
  whatever the accumulation order and are compared bit for bit, on every kernel instantiation (asserted with torch.profiler), every
  store path (TMA store; the 5-D strided TMA store of a ConvTranspose2d with cout % 32 == 0; the per-thread stores otherwise) and
  the tile edges, with the output written into a sentinel-filled wider tensor plus one spare frame;
- the production calls: every ops.conv2d / ops.deconv2d of one BaseBEVBackbone + CenterHead forward on the Waymo BEV map (188 x 188
  x 256) at batch 1 and the benchmark's batch 8, on their real operands and again with the input pixels rescaled by 10^U(-3, 3),
  against the element-wise bound spconv_arith.bound()."""
import inspect

import pytest
import torch

from tests import spconv_arith as sa
from tests import util
from detzero_b200 import _lib, ops, synthetic

pytestmark = pytest.mark.gpu
F64 = torch.float64
MODES = {'fp32': _lib.DZ_F32, 'tf32': _lib.DZ_TF32}
SENTINEL = -777.25
INSTANTIATIONS = ['k_conv2d_tf32<32, false>', 'k_conv2d_tf32<64, false>', 'k_conv2d_tf32<128, false>',
                  'k_conv2d_tf32<32, true>', 'k_conv2d_tf32<64, true>', 'k_conv2d_tf32<128, true>',
                  'k_conv2d_tf32_halo_n256<64>', 'k_conv2d_tf32_halo_n256<128>',
                  'k_conv2d_f32<128, 8>', 'k_conv2d_f32<64, 4>', 'k_conv2d_f32<16, 1>']


# ---------------------------------------------------------------------------------------------------------------------------------
# exact operands, bit for bit
# ---------------------------------------------------------------------------------------------------------------------------------
# (id, mode, transposed, cin, cout, k (deconv: s), stride, pad, H, W, B, coff, cstride, relu, scale, kernel, store).  The tile counts
# against DZ_NUM_SMS = 132 that pick each kernel (conv2d_tc.cu: halo_n256 needs cout >= 64 and >= 132 tiles of 32 x 8 (cout > 64)
# / 32 x 16 pixels; the 128-pixel halo kernel >= 264 tiles of 16 x 8 pixels x 128-channel tiles; else the generic kernel) are in the
# comments; the profiler assertion is the check.
CASES = [
    # generic 8 x 16 patches: stride 2 with odd input sizes, cin = 32 (one slice), cout 12 < 32 into a channel slice
    ('generic32_s2', 'tf32', False, 32, 12, 3, 2, 1, 37, 29, 3, 4, 20, True, True, 'k_conv2d_tf32<32, false>', 'tma'),
    # 3x3 stride 1 pad 0 with too few tiles for a halo kernel (2 x 3 x 2 = 12 patches), cout 36, no ReLU, no scale
    ('generic64_pad0', 'tf32', False, 64, 36, 3, 1, 0, 23, 21, 2, 0, 36, False, False, 'k_conv2d_tf32<64, false>', 'tma'),
    # 1x1 with cout 80 (a ragged 128-channel tile) at a channel offset
    ('generic128_1x1', 'tf32', False, 128, 80, 1, 1, 0, 30, 17, 2, 32, 160, True, True, 'k_conv2d_tf32<128, false>', 'tma'),
    # the BEV downsampling conv: stride 2 on odd sizes, two 128-channel tiles
    ('generic128_s2', 'tf32', False, 128, 256, 3, 2, 1, 47, 45, 2, 0, 256, True, True, 'k_conv2d_tf32<128, false>', 'tma'),
    # the CenterHead's last conv: 384 -> the padded head width 12, no ReLU, no scale; 6 x 13 x 5 = 390 patches
    ('halo32_head', 'tf32', False, 384, 12, 3, 1, 1, 100, 90, 5, 0, 12, False, False, 'k_conv2d_tf32<32, true>', 'tma'),
    # cin = 32, cout 36, pad 0: 5 x 9 x 7 = 315 patches
    ('halo64_pad0', 'tf32', False, 32, 36, 3, 1, 0, 67, 75, 7, 4, 44, True, True, 'k_conv2d_tf32<64, true>', 'tma'),
    # the CenterHead's shared conv at batch 1, cin = 512: 12 x 24 = 288 patches, 12 x 6 = 72 N=256 tiles
    ('halo64_cin512', 'tf32', False, 512, 64, 3, 1, 1, 188, 188, 1, 0, 64, True, True, 'k_conv2d_tf32<64, true>', 'tma'),
    # cout 80: 1 x 4 x 80 = 320 patches but 1 x 1 x 80 = 80 N=256 tiles; each 31 x 7 frame ends inside its tiles
    ('halo128_narrow', 'tf32', False, 128, 80, 3, 1, 1, 31, 7, 80, 16, 128, True, True, 'k_conv2d_tf32<128, true>', 'tma'),
    # 6 x 4 x 8 = 192 tiles of 32 x 16
    ('n256_64', 'tf32', False, 64, 64, 3, 1, 1, 100, 90, 8, 32, 160, True, True, 'k_conv2d_tf32_halo_n256<64>', 'tma'),
    # 10 x 3 x 8 = 240 tiles of 32 x 8, cout 80, no ReLU
    ('n256_128_ragged', 'tf32', False, 64, 80, 3, 1, 1, 70, 75, 8, 16, 128, False, True, 'k_conv2d_tf32_halo_n256<128>', 'tma'),
    # pad 0, three 128-channel tiles: 9 x 2 x 3 x 3 = 162 tiles
    ('n256_128_pad0', 'tf32', False, 256, 384, 3, 1, 0, 63, 69, 3, 0, 384, True, True, 'k_conv2d_tf32_halo_n256<128>', 'tma'),
    # ConvTranspose2d(kernel = stride): 2 x 2 with cout % 32 == 0 through the 5-D TMA store (odd H), else per-thread stores; 1 x 1
    ('deconv_s2_tma5d', 'tf32', True, 64, 64, 2, 2, 0, 7, 9, 3, 32, 128, True, True, 'k_conv2d_tf32<128, false>', 'tma5d'),
    ('deconv_s2_store36', 'tf32', True, 128, 36, 2, 2, 0, 11, 20, 1, 4, 44, True, True, 'k_conv2d_tf32<128, false>', 'thread'),
    ('deconv_s2_store4', 'tf32', True, 32, 4, 2, 2, 0, 5, 6, 2, 0, 4, False, False, 'k_conv2d_tf32<32, false>', 'thread'),
    ('deconv_s2_bev', 'tf32', True, 256, 256, 2, 2, 0, 13, 11, 2, 256, 512, True, True, 'k_conv2d_tf32<128, false>', 'tma5d'),
    ('deconv_s1_bev', 'tf32', True, 128, 256, 1, 1, 0, 13, 11, 2, 0, 512, True, True, 'k_conv2d_tf32<128, false>', 'tma'),
    # exact fp32
    ('f32_128', 'fp32', False, 64, 80, 3, 2, 1, 23, 19, 2, 8, 96, True, True, 'k_conv2d_f32<128, 8>', 'thread'),
    ('f32_64', 'fp32', False, 24, 36, 3, 1, 0, 13, 11, 3, 0, 36, False, True, 'k_conv2d_f32<64, 4>', 'thread'),
    ('f32_16_cin512', 'fp32', False, 512, 12, 3, 1, 1, 9, 10, 2, 0, 12, False, False, 'k_conv2d_f32<16, 1>', 'thread'),
    ('f32_deconv', 'fp32', True, 64, 12, 2, 2, 0, 7, 9, 2, 16, 28, True, True, 'k_conv2d_f32<16, 1>', 'thread'),
]


def test_cases_cover_every_instantiation_and_store_path():
    assert {c[15] for c in CASES} == set(INSTANTIATIONS)
    assert {c[16] for c in CASES if c[1] == 'tf32'} == {'tma', 'tma5d', 'thread'}


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_exact_operands_bit_exact(cuda, case):
    _, mode, transposed, cin, cout, k, stride, pad, H, W, B, coff, cstride, relu, has_scale, kernel, _ = case
    g = torch.Generator().manual_seed(sum(map(ord, case[0])))
    x, w, scale, shift = sa.exact_dense(g, mode, B, H, W, cin, cout, k, k, transposed)
    x, w, scale, shift = x.to(cuda), w.to(cuda), scale.to(cuda), shift.to(cuda)
    if not has_scale:
        scale = None
    sa.assert_exact_dense(mode, x, w, stride, pad, transposed)
    if transposed:
        Ho, Wo = H * k, W * k
    else:
        Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    buf = torch.full((B + 1, Ho, Wo, cstride), SENTINEL, device=cuda)                 # one spare frame past the output
    if transposed:
        wp = ops.pack_deconv_weight(w, MODES[mode])
        run = lambda: ops.deconv2d(x, wp, (k, cin, cout), scale, shift, relu, out=buf[:B], out_coff=coff, mode=MODES[mode])  # noqa: E731
    else:
        wp = ops.pack_conv_weight(w, MODES[mode])
        run = lambda: ops.conv2d(x, wp, (k, k, cin, cout), stride, pad, scale, shift, relu, out=buf[:B], out_coff=coff,  # noqa: E731
                                 mode=MODES[mode])
    _, seen = util.conv2d_kernels(run)
    assert seen == {kernel}, seen
    y, _ = sa.dense_contract64(mode, x, w, stride, pad, transposed)
    one = torch.ones(cout, device=cuda)
    o = sa.epilogue_exact(mode, y, one if scale is None else scale, shift, None, relu)
    assert torch.equal(o, o.float().to(F64)), 'the epilogue must be exact'
    util.assert_equal_signed(buf[:B, ..., coff:coff + cout], sa.output_bits(mode, o.float(), relu), case[0])
    assert bool((buf[:B, ..., :coff] == SENTINEL).all()) and bool((buf[:B, ..., coff + cout:] == SENTINEL).all()), 'other channels'
    assert bool((buf[B] == SENTINEL).all()), 'the frame past the output'


# ---------------------------------------------------------------------------------------------------------------------------------
# the production calls of BaseBEVBackbone + CenterHead, element by element
# ---------------------------------------------------------------------------------------------------------------------------------
def _bev_input(B, dev, seed=5):
    """a Waymo BEV map (B, 188, 188, 256) as HeightCompression leaves it in the default bf16x2 sparse mode: a quarter of the pixels
    occupied by ReLU outputs stored as plane 0 + plane 1 (not TF32-representable)"""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(B, 188, 188, 256, generator=g).clamp_min(0) * 2
    v = v * (torch.rand(B, 188, 188, 1, generator=g) < 0.25)
    p0, p1 = sa.split_bf16(v)
    return (p0 + p1).to(dev)


def _torch_weight(name, wp, kshape, mode):
    """the packed weight back in torch layout (tf32: it is RN(w), the weight the kernel multiplies)"""
    if name == 'conv2d':
        KH, KW, cin, cout = kshape
        return wp.view(cout, KH, KW, cin).permute(0, 3, 1, 2) if mode == _lib.DZ_TF32 else wp.view(KH, KW, cin, cout).permute(3, 2, 0, 1)
    s, cin, cout = kshape
    return wp.view(s, s, cout, cin).permute(3, 2, 0, 1) if mode == _lib.DZ_TF32 else wp.view(s, s, cin, cout).permute(2, 3, 0, 1)


def _wrap(mp, name, after):
    """replace ops.<name> by a wrapper that runs the kernel under the profiler and then calls after(orig, name, bound arguments,
    result, conv2d kernels that ran)"""
    orig = getattr(ops, name)
    sig = inspect.signature(orig)

    def wrapper(*args, **kwargs):
        out, kernels = util.conv2d_kernels(lambda: orig(*args, **kwargs))
        a = sig.bind(*args, **kwargs)
        a.apply_defaults()
        after(orig, name, a.arguments, out, kernels)
        return out
    mp.setattr(ops, name, wrapper)


@pytest.mark.parametrize('mode,B', [('tf32', 1), ('tf32', 8), ('fp32', 1)])
def test_bev_backbone_and_head_calls_elementwise(cuda, mode, B, monkeypatch):
    from detzero_b200.det import cp_modules
    cfg = synthetic.model_cfg(mode=mode)
    b2d = cp_modules['BaseBEVBackbone'](model_cfg=cfg.BACKBONE_2D, input_channels=256).eval()
    head = cp_modules['CenterHead'](model_cfg=cfg.DENSE_HEAD, input_channels=512, num_class=3, class_names=util.CLASS_NAMES,
                                    grid_size=[1504, 1504, 40], point_cloud_range=util.WAYMO_RANGE, voxel_size=util.VOXEL).eval()
    synthetic.load_seeded(b2d, 31)
    synthetic.load_seeded(head, 32)
    b2d, head = b2d.to(cuda), head.to(cuda)
    bev = _bev_input(B, cuda)
    g = torch.Generator(device=cuda).manual_seed(7)
    worst, calls = {}, []

    def check(orig, name, a, out, kernels):
        x, wp, kshape, m = a['x'], a['weight_packed'], a['kshape'], a['mode']
        smode = 'tf32' if m == _lib.DZ_TF32 else 'fp32'
        assert len(kernels) == 1, kernels
        kernel = kernels.pop()
        calls.append((name, tuple(x.shape), kshape, kernel))
        if smode == 'tf32' and x.data_ptr() != bev.data_ptr():
            assert sa.tf32_exact(x), 'a conv after the first must read a TF32-exact (RNA-rounded ReLU) input'
        transposed = name == 'deconv2d'
        stride, pad = (1, 0) if transposed else (a['stride'], a['pad'])
        w = _torch_weight(name, wp, kshape, m)
        cout = kshape[-1]
        coff = a['out_coff']
        what = '%s %s %s %s' % (name, tuple(x.shape), kshape, kernel)
        r = sa.assert_conv2d(out[..., coff:coff + cout], x, w, stride, pad, a['scale'], a['shift'], a['relu'], smode, what, transposed)
        worst[(kernel, 'collected')] = max(worst.get((kernel, 'collected'), 0.0), r)
        # the same call with every input pixel scaled by 10^U(-3, 3), still TF32-exact where the input was: small outputs on their
        # own scale
        f = torch.pow(10.0, torch.rand(x.shape[:3] + (1,), generator=g, device=cuda) * 6 - 3)
        xs = x * f
        if smode == 'tf32' and sa.tf32_exact(x):
            xs = ops.round_tf32(xs)
        buf = torch.full_like(out, SENTINEL)
        kw = dict(a)
        kw.update(x=xs, out=buf)
        orig(**kw)
        r = sa.assert_conv2d(buf[..., coff:coff + cout], xs, w, stride, pad, a['scale'], a['shift'], a['relu'], smode,
                             what + ' rescaled', transposed)
        assert bool((buf[..., :coff] == SENTINEL).all()) and bool((buf[..., coff + cout:] == SENTINEL).all())
        worst[(kernel, 'rescaled')] = max(worst.get((kernel, 'rescaled'), 0.0), r)

    _wrap(monkeypatch, 'conv2d', check)
    _wrap(monkeypatch, 'deconv2d', check)
    with torch.no_grad():
        d = b2d({'spatial_features': bev.permute(0, 3, 1, 2)})
        d['batch_size'] = B
        head(d)
    torch.cuda.synchronize()
    assert len(calls) == 17, calls       # 6 + 6 block convs, 2 deblocks, the shared conv, the two fused head stages
    assert calls[0][1] == tuple(bev.shape)
    print('\n%s B=%d: largest err/bound per kernel' % (mode, B))
    for (kernel, kind), v in sorted(worst.items()):
        print('  %-32s %-9s %.3g' % (kernel, kind, v))


def test_misaligned_base_pointers_are_refused(cuda):
    """a view at an odd storage offset: the fp32 kernel's float4 input loads and the tensor-core per-thread float2 stores need 16- and
    8-byte aligned base pointers; the entry points refuse such tensors instead of faulting"""
    B, H, W, cin, cout = 1, 8, 16, 32, 36
    w = torch.randn(cout, cin, 3, 3, device=cuda)
    wd = torch.randn(cin, cout, 2, 2, device=cuda)
    x = torch.randn(B, H, W, cin, device=cuda)
    x_odd = torch.empty(B * H * W * cin + 1, device=cuda)[1:].view(B, H, W, cin)
    x_odd.copy_(x)
    for mode in (_lib.DZ_F32, _lib.DZ_TF32):
        with pytest.raises(RuntimeError, match='bad argument'):
            ops.conv2d(x_odd, ops.pack_conv_weight(w, mode), (3, 3, cin, cout), 1, 1, None, None, True, mode=mode)
        with pytest.raises(RuntimeError, match='bad argument'):
            ops.deconv2d(x_odd, ops.pack_deconv_weight(wd, mode), (2, cin, cout), None, None, True, mode=mode)
        out_odd = torch.empty(B * H * W * cout + 1, device=cuda)[1:].view(B, H, W, cout)
        with pytest.raises(RuntimeError, match='bad argument'):
            ops.conv2d(x, ops.pack_conv_weight(w, mode), (3, 3, cin, cout), 1, 1, None, None, True, out=out_odd, mode=mode)
        dout_odd = torch.empty(B * 2 * H * 2 * W * cout + 1, device=cuda)[1:].view(B, 2 * H, 2 * W, cout)
        with pytest.raises(RuntimeError, match='bad argument'):
            ops.deconv2d(x, ops.pack_deconv_weight(wd, mode), (2, cin, cout), None, None, True, out=dout_odd, mode=mode)
        # the aligned tensors run
        ops.conv2d(x, ops.pack_conv_weight(w, mode), (3, 3, cin, cout), 1, 1, None, None, True, mode=mode)
    torch.cuda.synchronize()

"""The N=256 halo conv2d kernel (3x3 stride-1, output channels on the wgmma M side, 256-pixel patches on N) element by element
against float64 (spconv_arith.assert_conv2d):
every channel-tile width it takes, ragged image edges and channel tiles, output at a channel offset of a wider tensor, and frame
independence of a batch."""
import pytest
import torch

from tests import spconv_arith as sa
from tests import util
from detzero_b200 import _lib, ops

pytestmark = pytest.mark.gpu


def _nhwc(cuda, x):
    return x.permute(0, 2, 3, 1).contiguous().to(cuda)


def _inputs(seed, B, cin, cout, H, W):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, 3, 3, generator=g) * 0.05
    scale, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1
    return x, w, scale, shift


def _conv(cuda, x, w, scale, shift, cin, cout, out=None, coff=0):
    return ops.conv2d(_nhwc(cuda, x), ops.pack_conv_weight(w, _lib.DZ_TF32).to(cuda), (3, 3, cin, cout), 1, 1,
                      scale.to(cuda), shift.to(cuda), True, out=out, out_coff=coff, mode=_lib.DZ_TF32)


# (cin, cout, H, W, B, coff, cstride): H and W multiples of neither 32 nor 8, batch sizes that give at least one 256-pixel tile per SM;
# cout 64 (64-channel tiles over 32 x 16 patches), 80 (a ragged 128-channel tile with a partial 32-channel store), 128, 256, 384
@pytest.mark.parametrize('cin,cout,H,W,B,coff,cstride', [(64, 64, 100, 90, 6, 32, 160), (64, 80, 70, 75, 8, 16, 128),
                                                          (64, 128, 61, 67, 8, 128, 384), (128, 256, 45, 37, 8, 0, 256),
                                                          (64, 384, 95, 93, 4, 32, 448)])
def test_conv2d_halo_n256(cuda, cin, cout, H, W, B, coff, cstride):
    x, w, scale, shift = _inputs(17, B, cin, cout, H, W)
    out = torch.full((B, H, W, cstride), -3.0, device=cuda)
    _, seen = util.conv2d_kernels(lambda: _conv(cuda, x, w, scale, shift, cin, cout, out=out, coff=coff))
    assert seen == {'k_conv2d_tf32_halo_n256<%d>' % (128 if cout > 64 else 64)}, ('the shape did not select the N=256 halo kernel', seen)
    sa.assert_conv2d(out[..., coff:coff + cout], _nhwc(cuda, x), w, 1, 1, scale, shift, True, 'tf32', 'halo n256')
    assert torch.all(out[..., :coff] == -3.0) and torch.all(out[..., coff + cout:] == -3.0)


def test_conv2d_halo_n256_frames_independent(cuda):
    """frame b of a batch is bit-equal to that frame run alone: no tile reads across a frame boundary (each frame alone still
    has enough tiles for the N=256 kernel)"""
    cin, cout, H, W, B = 128, 128, 187, 181, 3
    x, w, scale, shift = _inputs(23, B, cin, cout, H, W)
    both = _conv(cuda, x, w, scale, shift, cin, cout)
    for b in range(B):
        one = _conv(cuda, x[b:b + 1], w, scale, shift, cin, cout)
        assert torch.equal(both[b:b + 1], one), b

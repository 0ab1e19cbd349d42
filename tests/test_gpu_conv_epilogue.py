"""GPU tests for the tensor-core conv beyond test_gpu_det.py: ConvTranspose2d(kernel = stride = 2) as one GEMM over all
four sub-pixels, with odd output rows through the strided TMA store and a cout that is not a multiple of 32 through the
per-thread stores."""
import pytest
import torch

from tests import spconv_arith as sa
from detzero_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('B,cin,cout,H,W,coff,ctot', [(2, 64, 64, 7, 9, 0, 64), (1, 128, 36, 11, 20, 4, 44), (3, 32, 256, 5, 47, 256, 512)])
def test_deconv2d_tf32_one_gemm(cuda, B, cin, cout, H, W, coff, ctot):
    from detzero_b200 import ops
    g = torch.Generator().manual_seed(B * H + W)
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cin, cout, 2, 2, generator=g) * 0.05
    scale, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1
    out = torch.full((B, 2 * H, 2 * W, ctot), -3.0, device=cuda)
    n0 = ops.launch_count()
    xh = x.permute(0, 2, 3, 1).contiguous().to(cuda)
    ops.deconv2d(xh, ops.pack_deconv_weight(w, _lib.DZ_TF32).to(cuda), (2, cin, cout), scale.to(cuda),
                 shift.to(cuda), True, out=out, out_coff=coff, mode=_lib.DZ_TF32)
    assert ops.launch_count() - n0 == 1
    sa.assert_conv2d(out[..., coff:coff + cout], xh, w, 1, 0, scale, shift, True, 'tf32', 'deconv', transposed=True)
    assert torch.all(out[..., :coff] == -3.0) and torch.all(out[..., coff + cout:] == -3.0)

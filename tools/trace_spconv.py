"""Clock trace of one CTA of the tensor-core sparse conv (64->64 SubM, ~35 K sites): who waits on whom in the
producer -> wgmma pipeline.  usage: [DZ_SPCONV_PW=1|2] python tools/trace_spconv.py"""
import ctypes, numpy as np, torch, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detzero_b200 import ops, _lib
from detzero_b200.spconv.pytorch import SparseConvTensor
from oracle import weights
l = ctypes.CDLL(_lib.LIB_PATH)
l.dz_debug_trace.argtypes = [ctypes.c_void_p, ctypes.c_int]
buf = np.zeros(4096, np.int64)
l.dz_debug_trace(buf.ctypes.data, 4096)     # allocate + switch the trace on
dev = torch.device('cuda')
shape, B = [5, 188, 188], 1
idx = weights.random_sparse_coords(1, B, shape, 0.2)       # ~35K sites dense-ish
f = torch.randn(len(idx), 64)
t = SparseConvTensor(f.to(dev), torch.from_numpy(idx).to(dev), shape, B)
nbr = ops.rulebook_subm(t._idx, t._count, t._cap, t.grid_index(), [3, 3, 3], layout="row")
w = torch.randn(64, 3, 3, 3, 64) * 0.05
wp = ops.pack_spconv_weight(w, _lib.DZ_TF32).to(dev)
for _ in range(3):
    out = ops.spconv_fwd(t._feat, nbr, t._count, len(idx), wp, None, None, None, True, _lib.DZ_TF32, kshape=(27, 64, 64))
torch.cuda.synchronize()
l.dz_debug_trace(buf.ctypes.data, 4096)
t0, t1, nb, t3, t4 = buf[0], buf[1], buf[2], buf[3], buf[4]
print('PW', os.environ.get('DZ_SPCONV_PW', 'default'), 'n sites', len(idx), 'nb', nb, 'prologue', t1 - t0, 'mainloop', t3 - t1, 'epilogue', t4 - t3,
      'total', t4 - t0, 'cycles')
n = int(min(nb, 120))
st = buf[8:8 + 8 * n].reshape(-1, 8)[:, :6] - t0
print('it: producer[wait_empty_start, empty_ok, issued]  mma[wait_full_start, full_ok, committed]')
for i in range(min(n, 16)):
    print(i, st[i].tolist())
print('per k-step (steady state, it >= 8): full_ok delta mean %.0f | producer: wait-for-empty %.0f, issue %.0f | data lands %.0f after issue | '
      'mma: wait-for-full %.0f, issue+commit %.0f' % (
          np.diff(st[8:, 4]).mean(), (st[8:, 1] - st[8:, 0]).mean(), (st[8:, 2] - st[8:, 1]).mean(), (st[8:, 4] - st[8:, 2]).mean(),
          (st[8:, 4] - st[8:, 3]).mean(), (st[8:, 5] - st[8:, 4]).mean()))

"""time one dense BEV conv (default 128->128 3x3 at 188x188) through the C ABI"""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detzero_b200 import ops, _lib
cin, cout, hw = [int(v) for v in (sys.argv[1:4] + [128, 128, 188][len(sys.argv) - 1:])][:3]
dev = torch.device('cuda')
NB = int(os.environ.get('BATCH', 1))
x = torch.randn(NB, hw, hw, cin, device=dev)
w = ops.pack_conv_weight(torch.randn(cout, cin, 3, 3) * 0.05, _lib.DZ_TF32).to(dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
ts = []
for i in range(13):
    if not os.environ.get('WARM'):
        flush.zero_()
    else:
        y = ops.conv2d(x, w, (3, 3, cin, cout), 1, 1, None, None, True, mode=_lib.DZ_TF32)      # same-config predecessor, warm L2
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    y = ops.conv2d(x, w, (3, 3, cin, cout), 1, 1, None, None, True, mode=_lib.DZ_TF32)
    e1.record()
    torch.cuda.synchronize()
    if i >= 3: ts.append(e0.elapsed_time(e1) * 1000)
ts.sort()
fl = 2.0 * NB * hw * hw * cin * cout * 9
print('batch %d conv %d->%d 3x3 @%d^2: median %.1f us  (%.0f TFLOP/s)' % (NB, cin, cout, hw, ts[len(ts) // 2], fl / ts[len(ts) // 2] / 1e6))
# steady state: a CUDA graph of 10 back-to-back convs (x -> y -> x ...): no host latency, warm L2, real launch gaps
if cin == cout:
    y = torch.empty_like(x)
    sgr = torch.cuda.Stream()
    with torch.cuda.stream(sgr):
        for _ in range(2):
            ops.conv2d(x, w, (3, 3, cin, cout), 1, 1, None, None, True, out=y, mode=_lib.DZ_TF32)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for k in range(5):
                ops.conv2d(x, w, (3, 3, cin, cout), 1, 1, None, None, True, out=y, mode=_lib.DZ_TF32)
                ops.conv2d(y, w, (3, 3, cin, cout), 1, 1, None, None, True, out=x, mode=_lib.DZ_TF32)
    tg = []
    for i in range(8):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
        tg.append(e0.elapsed_time(e1) * 100)
    tg.sort()
    print('  back-to-back in a CUDA graph (10 convs): %.1f us per conv (%.0f TFLOP/s)' % (tg[len(tg) // 2], fl / tg[len(tg) // 2] / 1e6))

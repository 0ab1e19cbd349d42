"""Per-kernel time of one warmed-up eager step of the bench workload (config 2), measured with torch.profiler (CUDA activity).

    python tools/profile_frame.py [--json OUT.json]

Prints every kernel of the step with its summed device time and launch count, then every dense conv2d / deconv2d call of
the BEV backbone and CenterHead in launch order with its FLOP (from the shapes), device time and TFLOP/s against the H100
SXM data-sheet TF32 peak (495 TFLOP/s dense).  Tracing slows the host, so these are kernel times, not bench values."""
import argparse
import json
import os
import sys
from collections import OrderedDict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

import bench
from detzero_b200 import ops
from detzero_b200 import synthetic as weights
from detzero_b200.det.centerpoint import build_network

TF32_PEAK = 495.0           # TFLOP/s, H100 SXM data sheet, dense


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--json', default=None, help='also write the tables here')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'profile_frame.py needs a GPU'
    sp_mode = os.environ.get('DZ_SP_MODE', weights.DEFAULT_SP_MODE)
    dev = torch.device('cuda', 0)
    batch = int(os.environ.get('DZ_BATCH', '8'))
    ds, batches = bench.build_inputs(batch)
    model = build_network(bench.make_model_cfg('VoxelBackBone8x', 'tf32', sp_mode), 3, ds).eval()
    weights.load_seeded(model, 3)
    bench.tune_head_for_bench(model)
    model = model.to(dev)
    pts = [torch.from_numpy(b['points']).to(dev) for b in batches]

    def bd(i):
        b = batches[i % len(batches)]
        return {'points': pts[i % len(batches)], 'points_per_frame': b['points_per_frame'], 'frame_id': b['frame_id'],
                'batch_size': b['batch_size']}

    # dense conv calls in launch order: (label, FLOP, kernel launches), recorded by wrapping the ops entry points
    calls = []
    conv2d, deconv2d = ops.conv2d, ops.deconv2d

    def conv2d_rec(x, w, kshape, stride, pad, *a, **k):
        n0 = ops.launch_count()
        out = conv2d(x, w, kshape, stride, pad, *a, **k)
        KH, KW, cin, cout = kshape
        B, Ho, Wo = out.shape[:3]
        calls.append(('conv %dx%d s%d %d->%d @%dx%d' % (KH, KW, stride, cin, cout, Ho, Wo),
                      2.0 * B * Ho * Wo * cout * KH * KW * cin, ops.launch_count() - n0))
        return out

    def deconv2d_rec(x, w, kshape, *a, **k):
        n0 = ops.launch_count()
        out = deconv2d(x, w, kshape, *a, **k)
        s, cin, cout = kshape
        B, H, W = x.shape[:3]
        calls.append(('deconv k%d s%d %d->%d @%dx%d' % (s, s, cin, cout, H, W), 2.0 * B * H * W * s * s * cout * cin,
                      ops.launch_count() - n0))
        return out

    with torch.no_grad():
        for _ in range(2):
            for i in range(len(batches)):
                model(bd(i))
        torch.cuda.synchronize()
        ops.conv2d, ops.deconv2d = conv2d_rec, deconv2d_rec
        try:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                model.forward_device(bd(0))
                torch.cuda.synchronize()
        finally:
            ops.conv2d, ops.deconv2d = conv2d, deconv2d

    kern = sorted((e for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA
                   and e.duration_ns() > 0 and not e.name().startswith('Memcpy') and not e.name().startswith('Memset')),
                  key=lambda e: e.start_ns())
    span_ms = (kern[-1].end_ns() - kern[0].start_ns()) / 1e6
    total_ms = sum(e.duration_ns() for e in kern) / 1e6
    per = OrderedDict()
    for e in kern:
        name = e.name()
        t, n = per.get(name, (0.0, 0))
        per[name] = (t + e.duration_ns() / 1e6, n + 1)
    print('one eager step, batch %d: %d kernels, %.3f ms kernel time, %.3f ms first start -> last end'
          % (batch, len(kern), total_ms, span_ms))
    print('%10s %6s %6s  %s' % ('ms', '%', 'calls', 'kernel'))
    rows = sorted(per.items(), key=lambda kv: -kv[1][0])
    for name, (t, n) in rows:
        print('%10.3f %6.1f %6d  %s' % (t, 100 * t / total_ms, n, name[:110]))

    # the dense conv kernels, matched to the recorded calls in launch order
    conv_k = [e for e in kern if 'k_conv2d_tf32' in e.name()]
    assert len(conv_k) == sum(c[2] for c in calls), (len(conv_k), sum(c[2] for c in calls))
    print('\ndense conv calls (TF32 peak %.0f TFLOP/s, H100 SXM data sheet)' % TF32_PEAK)
    print('%-40s %7s %9s %9s %6s %7s' % ('call', 'GFLOP', 'us', 'TFLOP/s', '%peak', 'launch'))
    conv_rows, i, conv_ms = [], 0, 0.0
    for label, flop, nl in calls:
        t = sum(e.duration_ns() for e in conv_k[i:i + nl]) / 1e6
        i += nl
        conv_ms += t
        tf = flop / (t * 1e-3) / 1e12
        conv_rows.append({'call': label, 'gflop': flop / 1e9, 'ms': t, 'tflops': tf, 'launches': nl})
        print('%-40s %7.1f %9.1f %9.1f %6.1f %7d' % (label, flop / 1e9, t * 1e3, tf, 100 * tf / TF32_PEAK, nl))
    conv_gflop = sum(c[1] for c in calls) / 1e9
    print('dense convs: %d calls, %d launches, %.3f ms = %.1f %% of kernel time, %.0f GFLOP issued, %.1f TFLOP/s'
          % (len(calls), len(conv_k), conv_ms, 100 * conv_ms / total_ms, conv_gflop, conv_gflop / conv_ms))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump({'device': torch.cuda.get_device_name(0), 'batch': batch, 'kernel_ms': total_ms, 'span_ms': span_ms,
                       'kernels': [{'name': n, 'ms': t, 'calls': c} for n, (t, c) in rows],
                       'conv_calls': conv_rows, 'conv_ms': conv_ms}, f, indent=1)


if __name__ == '__main__':
    main()

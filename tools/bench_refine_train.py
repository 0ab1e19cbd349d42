"""CRM training step on the device: the vehicle CRM config (vehicle_crm_model.yaml: ENCODER_MLP [128, 128], REGRESSION_MLP [512],
SCORE_THRESH [0.35, 0.7]), 200 boxes of 256 points of 32 features per track, B tracks per step, one step = forward + backward + Adam.

Reports tracks/s (best of N after warm-up, CUDA events), the device time of each point pass (torch.profiler, a separate run), the
peak memory, and the TFLOP/s those passes reach with FLOPs counted from the shapes of the passes that run.  Next to it, plain PyTorch
autograd of the same module tree in float32 (cuDNN TF32 allowed, as the reference trains) at B <= 64, for its peak memory per
track; that path is not run at B = 256."""
import argparse
import json
import os
import re
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detzero_b200.config import AttrDict  # noqa: E402
from detzero_b200.refine.modules import RefineTemplate  # noqa: E402
from detzero_b200.synthetic import crm_cfg, load_seeded  # noqa: E402

L, P, C0 = 200, 256, 32


def pass_macs_per_row(c0=C0):
    l1, l2, l3 = c0 * 128, 128 * 128, 128 * 256
    fwd = {1: l1, 2: l1 + l2, 3: l1 + l2 + l3, 4: l1 + l2 + l3}
    b5 = l1 + l2 + 6 * l3 + l2                 # L3 / L4 again, their dW, dy2, z2 again
    b6 = l1 + l2 + 4 * l3 + l2 + 2 * l2 + l1   # ... dz2's dW2 and dy1, z1 again
    b7 = b6 - l2 + 128 * c0
    return {**fwd, 5: b5, 6: b6, 7: b7}


def model(mode):
    cfg = crm_cfg()
    cfg.COMPUTE_MODE = mode
    m = RefineTemplate(AttrDict({'NAME': 'ConfidenceRefineModel', 'QUERY_POINT_DIMS': C0, 'MEMORY_POINT_DIMS': C0, 'REGRESSION': cfg}))
    load_seeded(m.reg, 11)
    return m.cuda().train()


def batch(B):
    g = torch.Generator(device='cuda').manual_seed(B)
    pts = torch.randn(B, L, P, C0, device='cuda', generator=g)
    iou = torch.rand(B, L, device='cuda', generator=g)
    return {'conf_points': pts, 'iou': iou}


def device_step(m, opt, d):
    opt.zero_grad(set_to_none=True)
    ret, _, _ = m(d)
    ret['loss'].backward()
    opt.step()


def torch_step(m, opt, d):
    """the reference's forward (confidence_pointnet.py:80-104) on the same modules, plain autograd"""
    r = m.reg
    pts = d['conf_points'].permute(0, 3, 1, 2)
    inter = r.pts_encoder_1[:6](pts)
    f = r.pts_encoder_1[6:](inter)
    f = torch.cat([f.max(dim=3)[0].unsqueeze(-1).expand(-1, -1, -1, P), inter], dim=1)
    pool = r.pts_encoder_2(f).max(dim=3)[0]
    tap = r.pts_mlp(pool)
    out = r.regression_mlp(torch.cat([tap.max(dim=2)[0].unsqueeze(-1).expand(-1, -1, L), tap], dim=1))
    preds = [torch.sigmoid(r.heads[t](out)).reshape(-1) for t in ('score_reg', 'iou_reg')]
    lab = d['iou'].clamp(0, 1).reshape(-1)
    loss = F.binary_cross_entropy(preds[0], (lab >= 0.7).float()) + F.binary_cross_entropy(preds[1], lab)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    best = float('inf')
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


def pass_times(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        mm = re.search(r'k_crm_point<\(?(\d)\)?, \(?(\d)\)?>', e.key)
        if mm:
            out[int(mm.group(2))] = out.get(int(mm.group(2)), 0.0) + e.device_time_total / 1e3 / max(e.count, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', default='64,256')
    ap.add_argument('--modes', default='tf32,fp32')
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--torch-batches', default='16,64')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_refine_train: needs a CUDA device (there is no CPU measurement)')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    macs = pass_macs_per_row()
    res = {'card': card, 'device': {}, 'torch_autograd': {}}
    for mode in args.modes.split(','):
        for B in [int(b) for b in args.batches.split(',')]:
            m = model(mode)
            opt = torch.optim.Adam(m.parameters(), lr=1e-3)
            d = batch(B)
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            ms = timed(lambda: device_step(m, opt, d), args.steps, args.warmup)
            peak = torch.cuda.max_memory_allocated()
            pt = pass_times(lambda: device_step(m, opt, d))
            rows = B * L * P
            tflops = {p: 2 * macs[p] * rows / (t * 1e-3) / 1e12 for p, t in pt.items()}
            res['device']['%s_B%d' % (mode, B)] = {
                'step_ms': round(ms, 2), 'tracks_per_s': round(B / (ms * 1e-3), 1), 'peak_GB': round(peak / 2**30, 2),
                'peak_above_inputs_GB': round((peak - base) / 2**30, 2), 'input_GB': round(d['conf_points'].numel() * 4 / 2**30, 2),
                'pass_ms': {p: round(t, 2) for p, t in sorted(pt.items())}, 'pass_tflops': {p: round(v, 1) for p, v in sorted(tflops.items())},
                'point_pass_share': round(sum(pt.values()) / ms, 3)}
            print(json.dumps({mode + '_B%d' % B: res['device']['%s_B%d' % (mode, B)]}), flush=True)
            del m, opt, d
            torch.cuda.empty_cache()
    torch.backends.cudnn.allow_tf32 = True
    for B in [int(b) for b in args.torch_batches.split(',')]:
        assert B <= 64
        m = model('tf32')
        opt = torch.optim.Adam(m.parameters(), lr=1e-3)
        d = batch(B)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        ms = timed(lambda: torch_step(m, opt, d), args.steps, args.warmup)
        peak = torch.cuda.max_memory_allocated() - base
        res['torch_autograd']['B%d' % B] = {'step_ms': round(ms, 2), 'tracks_per_s': round(B / (ms * 1e-3), 1),
                                            'peak_above_inputs_GB': round(peak / 2**30, 2), 'GB_per_track': round(peak / B / 2**30, 3),
                                            'B256_extrapolated_GB': round(peak / B * 256 / 2**30, 1)}
        print(json.dumps({'torch_B%d' % B: res['torch_autograd']['B%d' % B]}), flush=True)
        del m, opt, d
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()

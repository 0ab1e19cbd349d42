"""PRM training step on the device: the vehicle PRM config (vehicle_prm_model.yaml: QUERY_ENCODER / MEMORY_ENCODER [128, 128],
REGRESSION_MLP [512], EMBED_DIMS 256, one decoder layer), L = 200 box slots of 256 query and 48 memory points of 32 features per
track, B tracks per step, one step = forward + backward + Adam.

Reports tracks/s (best of N after warm-up, CUDA events), the peak memory, the device time of each forward part (query encoder +
query MLP, memory path, decoder + heads, loss; CUDA events around each, in a run of their own), of the backward and of Adam, and
the point-layer kernels' device time (torch.profiler, a separate run) with the TFLOP/s they reach, FLOPs counted from the shapes.
Next to it, in the same call, plain PyTorch autograd of the reference's module tree on the same modules (tests/prm_train_ref.py:
float32, TF32 matmuls and convolutions allowed, as the reference trains), at every B where it fits."""
import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detzero_b200.config import AttrDict  # noqa: E402
from detzero_b200.refine import train  # noqa: E402
from detzero_b200.refine.modules import RefineTemplate, _train_mlp  # noqa: E402
from detzero_b200.synthetic import load_seeded, prm_cfg  # noqa: E402
from tests import prm_train_ref as PR  # noqa: E402

L, P, PM, C = 200, 256, 48, 32


def macs_per_row():
    """multiply-adds per row of each kernel family: query encoder (per query point) and memory path (per memory point)"""
    q_fwd = C * 128 + 128 * 128 + 128 * 256
    mem_fwd = C * 128 + 128 * 128 + 128 * 256 + 128 * 512 + 512 * 256       # 384 -> 512 as a 128 -> 512 GEMM + a per-track shift
    q_dgrad = 256 * 128 + 128 * 128
    mem_dgrad = 256 * 512 + (512 + 256) * 128 + 128 * 128
    return {'k_pm_fwd': (q_fwd, mem_fwd), 'k_pm_dgrad': (q_dgrad, mem_dgrad), 'k_pm_wgrad': (q_fwd, mem_fwd)}


def model(mode):
    cfg = prm_cfg()
    cfg.COMPUTE_MODE = mode
    m = RefineTemplate(AttrDict({'NAME': 'PositionRefineModel', 'QUERY_POINT_DIMS': C, 'MEMORY_POINT_DIMS': C, 'REGRESSION': cfg}))
    load_seeded(m.reg, 11)
    return m.cuda().train()


def batch(B):
    """B tracks, box_num uniform on 1..L, padded boxes zero rows"""
    g = torch.Generator(device='cuda').manual_seed(B)
    box_num = torch.from_numpy(np.random.default_rng(B).integers(1, L + 1, B).astype(np.int32)).cuda()
    valid = torch.arange(L, device='cuda')[None] < box_num[:, None]
    traj = torch.randn(B, L, 7, device='cuda', generator=g)
    traj[..., 3:6] = torch.tensor([4.5, 1.9, 1.6], device='cuda')
    gt = traj + 0.1 * torch.randn(B, L, 7, device='cuda', generator=g)
    v4 = valid[:, :, None, None]
    return {'pos_query_points': torch.randn(B, L, P, C, device='cuda', generator=g) * v4,
            'pos_memory_points': torch.randn(B, L, PM, C, device='cuda', generator=g) * v4,
            'pos_trajectory': traj * valid[..., None], 'gt_pos_trajectory': gt * valid[..., None], 'padding_mask': (~valid).float(),
            'box_num': box_num, 'pos_init_box': torch.zeros(B, 7, device='cuda')}


def device_step(m, opt, d):
    opt.zero_grad(set_to_none=True)
    ret, _, _ = m(dict(d))
    ret['loss'].backward()
    opt.step()


def torch_step(m, opt, d):
    opt.zero_grad(set_to_none=True)
    loss, _ = PR.forward_loss(m.reg, d, torch.float32)
    loss.backward()
    opt.step()


def parts(m, opt, d):
    """device time (ms) of each part of one step, CUDA events around each part"""
    r = m.reg
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(7)]
    opt.zero_grad(set_to_none=True)
    B = d['pos_query_points'].shape[0]
    ev[0].record()
    q = _train_mlp(r.query_mlp, train.prm_query(r, d['pos_query_points']))
    ev[1].record()
    mem = train.prm_memory(r, d['pos_memory_points'])
    ev[2].record()
    traj = d['pos_trajectory']
    preds = r.decoder.forward_train(q.view(B, L, -1), mem.view(B, L * PM, -1), torch.cat([traj[..., :3], traj[..., 6:]], -1),
                                    d['padding_mask'], PM)
    r.preds_dict.update({k: v.view(B, L, -1) for k, v in preds.items()})
    ev[3].record()
    r.targets_dict.update(r.target_assigner.encode_torch(d))
    loss, _ = r.get_loss({})
    ev[4].record()
    loss.backward()
    ev[5].record()
    opt.step()
    ev[6].record()
    torch.cuda.synchronize()
    names = ('query_encoder_and_mlp', 'memory_path', 'decoder_and_heads', 'loss', 'backward', 'adam')
    return {n: round(ev[i].elapsed_time(ev[i + 1]), 2) for i, n in enumerate(names)}


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


def kernel_times(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out, total = {}, 0.0
    for e in prof.key_averages():
        t = e.device_time_total / 1e3
        total += t
        mm = re.search(r'(k_pm_\w+)', e.key)
        if mm:
            out[mm.group(1)] = out.get(mm.group(1), 0.0) + t
    return out, total


def measure(step, m, d, steps, warmup):
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    step(m, opt, d)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ms = timed(lambda: step(m, opt, d), steps, warmup)
    peak = torch.cuda.max_memory_allocated()
    return opt, ms, peak, base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', default='32,96')
    ap.add_argument('--modes', default='tf32,fp32')
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_prm_train: needs a CUDA device (there is no CPU measurement)')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    macs = macs_per_row()
    res = {'card': card, 'device': {}, 'torch_autograd': {}}
    print(json.dumps({'card': card}), flush=True)
    for B in [int(b) for b in args.batches.split(',')]:
        d = batch(B)
        for mode in args.modes.split(','):
            m = model(mode)
            opt, ms, peak, base = measure(device_step, m, d, args.steps, args.warmup)
            part = parts(m, opt, d)
            kt, total = kernel_times(lambda: device_step(m, opt, d))
            rows = (B * L * P, B * L * PM)
            tflops = {k: 2 * (macs[k][0] * rows[0] + macs[k][1] * rows[1]) / (t * 1e-3) / 1e12 for k, t in kt.items() if k in macs}
            r = {'step_ms': round(ms, 2), 'tracks_per_s': round(B / (ms * 1e-3), 1), 'peak_GB': round(peak / 2**30, 2),
                 'peak_above_model_and_inputs_GB': round((peak - base) / 2**30, 2), 'part_ms': part,
                 'kernel_ms': {k: round(t, 2) for k, t in sorted(kt.items())},
                 'kernel_tflops': {k: round(v, 1) for k, v in sorted(tflops.items())}, 'profiled_step_device_ms': round(total, 2)}
            res['device']['%s_B%d' % (mode, B)] = r
            print(json.dumps({'%s_B%d' % (mode, B): r}), flush=True)
            del m, opt
            torch.cuda.empty_cache()
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
        try:
            m = model('tf32')
            opt, ms, peak, base = measure(torch_step, m, d, args.steps, args.warmup)
            r = {'step_ms': round(ms, 2), 'tracks_per_s': round(B / (ms * 1e-3), 1), 'peak_GB': round(peak / 2**30, 2),
                 'peak_above_model_and_inputs_GB': round((peak - base) / 2**30, 2)}
        except torch.OutOfMemoryError:
            r = {'out_of_memory': True}
        finally:
            torch.backends.cuda.matmul.allow_tf32 = False
        res['torch_autograd']['B%d' % B] = r
        print(json.dumps({'torch_B%d' % B: r}), flush=True)
        m = opt = None
        del d
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == '__main__':
    main()

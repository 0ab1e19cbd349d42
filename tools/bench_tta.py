"""Measure CenterPoint test-time augmentation (15 views, device expansion + detector + un-augmentation + WBF) on the bench workload:
180 K-point synthetic Waymo frames, the default compute modes, the head tuned by bench.tune_head_for_bench so that every view
yields ~500 boxes.  Prints one JSON line per batch size:
  * TTA frames/s of a CUDA-graph replay, and the non-TTA frame rate of the same model and frames;
  * device time per stage from CUDA events (eager): expand, detector, un-augment, WBF;
  * boxes into and out of WBF;
  * the host oracle's WBF time on the same boxes (oracle/tta_ref.py, a numpy restatement -- not the reference's own code);
  * the card name and power limit.

    python tools/bench_tta.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown'


def build(tta):
    import bench
    from detzero_b200 import synthetic
    from detzero_b200.det import build_network
    from detzero_b200.det.dataset import SyntheticWaymoDataset, default_waymo_1sweep_cfg
    dcfg = default_waymo_1sweep_cfg()
    dcfg.TTA = tta
    ds = SyntheticWaymoDataset(dcfg, synthetic.CLASS_NAMES, training=False, num_frames=4, n_points=bench.N_POINTS)
    cfg = synthetic.model_cfg('VoxelBackBone8x', 'tf32')
    cfg.BACKBONE_3D.COMPUTE_MODE = synthetic.DEFAULT_SP_MODE
    model = build_network(cfg, 3, ds).eval()
    synthetic.load_seeded(model, 0)
    bench.tune_head_for_bench(model)
    return ds, model.cuda()


def graph_rate(model, batch, steps, warmup, frames):
    with torch.no_grad():
        for _ in range(warmup + 2):
            try:
                model(dict(batch))                               # settles the capacity hints
            except RuntimeError as e:                            # capacity overflow: the hints are raised, run again
                if 'capacity overflow' not in str(e):
                    raise
    g, out = model.capture_graph(dict(batch))
    for _ in range(warmup):
        g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return ms, frames * 1000.0 / ms, out


def stage_times(model, batch, reps):
    """eager device time of each TTA stage, CUDA events around each, averaged over `reps` runs"""
    from detzero_b200 import ops
    from detzero_b200.det import tta
    aug = tta.ops_from_names(batch['tta_ops'])
    ev, vw, uw = [], aug.expand_views(), aug.unaugment_views()
    V = len(aug)
    B = batch['batch_size'] // V
    acc = np.zeros(4)
    for _ in range(reps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        with torch.no_grad():
            ev[0].record()
            pts = ops.tta_expand(batch['points'], batch['points_per_frame'], vw)
            ev[1].record()
            inner = {k: v for k, v in batch.items() if k != 'tta_ops'}
            inner.update(points=pts, points_per_frame=[s for s in batch['points_per_frame'] for _ in range(V)], batch_size=B * V)
            for m in model.module_list:
                inner = m(inner)
            ev[2].record()
            un = ops.tta_unaugment(inner['final_boxes_padded'], inner['final_boxes_count'], uw)
            ev[3].record()
            fused, n = ops.wbf_3d(un, inner['final_boxes_count'], V, tta.WBF_IOU_THR, tta.WBF_SKIP_BOX_THR)
            ev[4].record()
        torch.cuda.synchronize()
        acc += [ev[i].elapsed_time(ev[i + 1]) for i in range(4)]
    return acc / reps, un, inner['final_boxes_count'], n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_tta.py measures on the GPU'
    from detzero_b200.det import load_data_to_gpu
    from oracle import tta_ref
    ds, model = build(True)
    plain_ds, _ = build(False)
    for B in (1, 2):
        items = [ds[i] for i in range(B)]
        batch = load_data_to_gpu(ds.collate_batch(items), 'cuda')
        V = len(batch['tta_ops'])
        ms, fps, _ = graph_rate(model, batch, args.steps, args.warmup, B)
        plain = load_data_to_gpu(plain_ds.collate_batch([plain_ds[i] for i in range(B)]), 'cuda')
        pms, pfps, _ = graph_rate(model, plain, args.steps, args.warmup, B)
        st, un, vcount, n = stage_times(model, batch, 5)
        vcount = vcount.cpu().numpy()
        u = un.cpu().numpy()
        K = u.shape[1]
        labels = np.where(np.arange(K)[None] < vcount[:V, None], u[:V, :, 8], 0).astype(np.int64)
        t0 = time.perf_counter()
        ref = tta_ref.wbf_3d(u[:V, :, :7], u[:V, :, 7], labels)
        host_ms = (time.perf_counter() - t0) * 1000
        print(json.dumps({
            'workload': 'CenterPoint TTA, %d views, %d x %dK-pt synthetic Waymo frame(s), CUDA graph' % (V, B, ds.n_points // 1000),
            'frames': B, 'tta_frames_per_s': round(fps, 2), 'tta_ms_per_step': round(ms, 3),
            'no_tta_frames_per_s': round(pfps, 2), 'no_tta_ms_per_step': round(pms, 3),
            'stage_ms': {'expand': round(st[0], 3), 'detector': round(st[1], 3), 'unaugment': round(st[2], 3), 'wbf': round(st[3], 3)},
            'wbf_boxes_in': int(vcount.sum()), 'wbf_boxes_out': n.cpu().tolist(),
            'host_oracle_wbf_ms_frame0': round(host_ms, 1), 'host_oracle_boxes_out_frame0': int(len(ref['scores'])),
            'card': card()}))


if __name__ == '__main__':
    main()

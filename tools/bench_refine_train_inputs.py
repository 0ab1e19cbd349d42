"""Refiner training samples on the device, per epoch, beside one step of each model.
Setup (not timed): the 199-frame sequence of tools/bench_offboard.py (180 K background points per frame, about 300 tracks of the
three classes), tracked (track.track_sequences) and assigned to its ground truth (track.assign_track_target, refine.data.track_targets),
with synthetic CRM IoU labels (uniform on [0, 1]: the builders only gather them).  Prints JSON lines with:
  * the card's name and power limit, read in the same run;
  * crop_tracks of every box once (CUDA events, best of --reps, after a warm-up);
  * per epoch, training_order plus every batch of each builder on the cropped rows (crop=False) at the shipped batch sizes (PRM
    B = 96, GRM B = 128, CRM B = 256): milliseconds and tracks/s (CUDA events around the epoch, host work included);
  * one device training step (forward, loss, backward) of the GRM and CRM in tf32 at the same B, on the first batch of the epoch;
    the PRM, which has no training step yet, gets its tf32 eval forward on that batch instead (prm_eval_forward_ms).
    python tools/bench_refine_train_inputs.py [--tracks 300] [--frames 199] [--background 180000] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detzero_b200 import synthetic                         # noqa: E402
from detzero_b200.config import AttrDict                   # noqa: E402
from detzero_b200.refine import data as D                  # noqa: E402
from detzero_b200.refine.modules import RefineTemplate     # noqa: E402
from detzero_b200.track import assign_track_target, ground_truth_from_infos, track_sequences            # noqa: E402
from oracle import refine_inputs as ri                     # noqa: E402
from oracle import weights                                 # noqa: E402


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [v.strip() for v in q.split(',')]
    except Exception:
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def _timed(fn, reps):
    best = None
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        t = e0.elapsed_time(e1)
        best = t if best is None else min(best, t)
    return best


def _model(kind):
    if kind == 'prm':
        c, spec = ri.prm_cfg(), {'NAME': 'PositionRefineModel', 'QUERY_POINT_DIMS': 32, 'MEMORY_POINT_DIMS': 32}
    elif kind == 'grm':
        c, spec = ri.grm_cfg(), {'NAME': 'GeometryRefineModel', 'QUERY_POINT_DIMS': 11, 'MEMORY_POINT_DIMS': 4}
    else:
        c, spec = ri.crm_cfg(), {'NAME': 'ConfidenceRefineModel', 'QUERY_POINT_DIMS': 32, 'MEMORY_POINT_DIMS': 32}
    c.COMPUTE_MODE = 'tf32'
    m = RefineTemplate(AttrDict(dict(spec, REGRESSION=c)))
    weights.load_seeded(m.reg, 1)
    return m.cuda().train()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--tracks', type=int, default=300)
    ap.add_argument('--frames', type=int, default=199)
    ap.add_argument('--background', type=int, default=180000)
    ap.add_argument('--radius', type=float, default=150.0)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--seed', type=int, default=1)
    ap.add_argument('--prm-batch', type=int, default=96)
    ap.add_argument('--grm-batch', type=int, default=128)
    ap.add_argument('--crm-batch', type=int, default=256)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_refine_train_inputs needs a GPU'
    dev = torch.device('cuda:0')
    card, power = _card()
    print(json.dumps({'card': card, 'power_limit': power}), flush=True)
    s = synthetic.synthetic_sequence(a.seed, frames=a.frames, tracks=a.tracks, n_background=a.background, ego_step=0.0, max_speed=0.3,
                                     radius=a.radius)
    boxes, counts, _ = synthetic.detections_from_sequence(s, a.seed)
    frames, poses = torch.from_numpy(s['frames']).to(dev), torch.from_numpy(s['poses']).to(dev)
    res = track_sequences(torch.from_numpy(boxes).to(dev), torch.from_numpy(counts).to(dev), poses, max_entries=1 << 20)
    gt = ground_truth_from_infos(synthetic.synthetic_ground_truth(s, a.seed), ['seq'], device=dev)
    tb = res.track_batch()
    tg = D.track_targets(assign_track_target(res, gt), tb)
    g = np.random.default_rng(a.seed)
    valid = torch.arange(tb.L, device=dev)[None, :] < tb.box_num[:, None]
    iou = torch.where(valid, torch.from_numpy(g.uniform(0, 1, (len(tb), tb.L)).astype(np.float32)).to(dev), -1.0)
    off = s['frame_offsets']

    crop = {}

    def do_crop():
        crop['out'] = D.crop_tracks(frames, off, poses, tb)
    do_crop()
    crop_ms = _timed(do_crop, a.reps)
    bf, bo, bp, btb = crop['out']
    print(json.dumps({'tracks': len(tb), 'boxes': int(tb.box_num.sum()), 'cropped_rows': int(bf.shape[0]),
                      'crop_tracks_ms': round(crop_ms, 3)}), flush=True)

    for kind, B in (('prm', a.prm_batch), ('grm', a.grm_batch), ('crm', a.crm_batch)):
        state = {'epoch': 0}

        def epoch():
            order = D.training_order(tg, kind, seed=a.seed, epoch=state['epoch'])
            first = None
            for i in range(0, len(order), B):
                idx = order[i:i + B].tolist()
                if kind == 'prm':
                    o = D.position_training_inputs(bf, bo, bp, btb.select(idx), tg.select(idx), seed=a.seed, epoch=state['epoch'],
                                                   crop=False)
                elif kind == 'grm':
                    o = D.geometry_training_inputs(bf, bo, bp, btb.select(idx), tg.select(idx), seed=a.seed, epoch=state['epoch'],
                                                   crop=False)
                else:
                    o = D.confidence_training_inputs(bf, bo, bp, btb.select(idx), iou[idx], seed=a.seed, epoch=state['epoch'],
                                                     crop=False)
                first = o if first is None else first
            state['epoch'] += 1
            state['n'], state['first'] = len(order), first
        epoch()
        ms = _timed(epoch, a.reps)
        m = _model(kind)
        batch = state['first'] if kind != 'crm' else {'conf_points': state['first']['conf_points'], 'iou': state['first']['iou']}
        nb = len(state['first']['geo_query_num' if kind == 'grm' else 'box_num'])
        row = {'kind': kind, 'batch': B, 'epoch_tracks': state['n'], 'epoch_ms': round(ms, 3),
               'tracks_per_s': round(state['n'] / ms * 1e3, 1), 'build_ms_per_batch': round(ms / max(1, -(-state['n'] // B)), 3)}
        if kind == 'prm':
            m.eval()

            def forward():
                with torch.no_grad():
                    m(dict(batch))
            forward()
            print(json.dumps(dict(row, prm_eval_forward_ms=round(_timed(forward, a.reps), 3), prm_eval_forward_batch=nb)), flush=True)
            continue

        def step():
            m.zero_grad(set_to_none=True)
            ret, _, _ = m(dict(batch))
            ret['loss'].backward()
        step()
        step_ms = _timed(step, a.reps)
        print(json.dumps(dict(row, train_step_ms=round(step_ms, 3), train_step_batch=nb)), flush=True)


if __name__ == '__main__':
    main()

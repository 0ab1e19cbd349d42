"""Throughput of Waymo AP / APH on the device (detzero_b200.evaluate, csrc/det_eval.cu): S in {1, 8} synthetic 199-frame sequences
with about 300 ground-truth objects and up to 500 predictions per frame (jittered detections of every object, shifted duplicates
of half of them, far false positives), breakdowns OBJECT_TYPE + RANGE, 3-D IoU.  Two calls are timed with CUDA events, best of
--reps after a warm-up: detection_metrics on the device tables (the kernel, its one device-to-host copy and the host AP), and
WaymoDetectionMetricsEstimator.waymo_evaluation from the frame dicts (host preparation and upload included).  Prints the card and
its power limit, one JSON line per S, and the numpy oracle's seconds per frame over the first --oracle-frames frames of one
sequence, for scale."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detzero_b200 import evaluate, synthetic                # noqa: E402
from detzero_b200.track import CLASS_NAMES                  # noqa: E402

CFG = ['object', 'range', '3d']


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    return min(times), times


def sequence(seed, F=199):
    """frame dicts (predictions, ground-truth annos) of one synthetic sequence"""
    s = synthetic.synthetic_sequence(seed, frames=F, tracks=600, n_background=100, max_pts=12, ego_step=0.5, max_speed=0.3,
                                     radius=75.0)
    gts = [i['annos'] for i in synthetic.synthetic_ground_truth(s, seed, name='seq%d' % seed)]
    boxes, counts, _ = synthetic.detections_from_sequence(s, seed, K=1000)
    g = np.random.default_rng([seed, 0xBE7])
    preds = []
    for f in range(F):
        rows = boxes[f, :counts[f]]
        dup = rows[g.random(len(rows)) < 0.5].copy()
        dup[:, 0] += g.uniform(-0.3, 0.3, len(dup))
        dup[:, 7] = g.uniform(0.02, 0.6, len(dup))
        rows = np.concatenate([rows, dup])[:500]
        preds.append({'boxes_lidar': rows[:, :7].copy(), 'score': rows[:, 7].copy(),
                      'name': np.array([CLASS_NAMES[int(c) - 1] for c in rows[:, 8]])})
    return preds, gts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='1,8')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--distinct', type=int, default=4)
    ap.add_argument('--oracle-frames', type=int, default=199)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_det_eval needs a GPU'
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print('card:', q.stdout.strip().splitlines()[0] if q.stdout else torch.cuda.get_device_name(0), flush=True)
    base = [sequence(100 + i) for i in range(a.distinct)]
    for S in [int(x) for x in a.sizes.split(',')]:
        preds = sum([base[i % len(base)][0] for i in range(S)], [])
        gts = sum([base[i % len(base)][1] for i in range(S)], [])
        est = evaluate.WaymoDetectionMetricsEstimator()
        t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda()
             for k, v in evaluate.frame_tables(preds, gts, CLASS_NAMES, 1000, False).items()}
        metrics = lambda: evaluate.detection_metrics(t['pred'], t['pred_cnt'], t['gt_box'], t['gt_type'], t['gt_level'], t['gt_cnt'],
                                                     '3d', ('object', 'range'))
        tm, all_m = timed(metrics, a.reps)
        tw, all_w = timed(lambda: est.waymo_evaluation(preds, gts, CLASS_NAMES, config_type=CFG, distance_thresh=1000,
                                                       fake_gt_infos=False), a.reps)
        rec, res = metrics()
        NF = len(preds)
        print(json.dumps({'S': S, 'frames': NF, 'gt_per_frame': float(t['gt_cnt'].float().mean()),
                          'pred_per_frame': float(t['pred_cnt'].float().mean()), 'metrics_seconds': tm, 'metrics_frames_per_s': NF / tm,
                          'waymo_evaluation_seconds': tw, 'waymo_evaluation_frames_per_s': NF / tw,
                          'vehicle_L2_APH': res['OBJECT_TYPE_TYPE_VEHICLE_LEVEL_2/APH'][0], 'metrics_all': all_m,
                          'waymo_evaluation_all': all_w}), flush=True)
    if a.oracle_frames > 0:
        from oracle import det_eval_ref
        n = a.oracle_frames
        t0 = time.time()
        det_eval_ref.waymo_evaluation(base[0][0][:n], base[0][1][:n], CLASS_NAMES, CFG, 1000, False)
        dt = time.time() - t0
        print(json.dumps({'oracle_frames': n, 'oracle_seconds_per_frame': dt / n}), flush=True)


if __name__ == '__main__':
    main()

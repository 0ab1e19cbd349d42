"""Throughput of the tracking MOTA / MOTP metric on the device (detzero_b200.evaluate, csrc/track_eval.cu): S in {1, 8, 64}
synthetic 199-frame sequences with 300 objects, their jittered detections tracked by track_sequences (4 distinct sequences,
repeated for S > 4), breakdowns OBJECT_TYPE + RANGE.  Two calls are timed with CUDA events, best of --reps after a warm-up:
evaluate_tracks on the TrackResult (the device table build, the kernel, its one device-to-host copy and the host dict) and
tracking_metrics on the prepared device tables.  Prints the card and its power limit, one JSON line per S, and the numpy oracle's
seconds per frame over the first --oracle-frames frames of one sequence, for scale.  This is launch-, latency- and
assignment-bound work; no share of a peak is claimed."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detzero_b200 import evaluate, synthetic                                       # noqa: E402
from detzero_b200.track import CLASS_NAMES, ground_truth_from_infos, track_sequences  # noqa: E402

CFG = ('object', 'range')


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='1,8,64')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--distinct', type=int, default=4)
    ap.add_argument('--oracle-frames', type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_track_eval needs a GPU'
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print('card:', q.stdout.strip().splitlines()[0] if q.stdout else torch.cuda.get_device_name(0), flush=True)
    F = 199
    base = []
    for seed in range(a.distinct):
        s = synthetic.synthetic_sequence(100 + seed, frames=F, tracks=300, n_background=200, ego_step=0.5, max_speed=0.3)
        boxes, counts, _ = synthetic.detections_from_sequence(s, 100 + seed)
        base.append((s, synthetic.synthetic_ground_truth(s, 100 + seed, name='seq%d' % seed), boxes, counts))
    for S in [int(x) for x in a.sizes.split(',')]:
        seqs = [base[i % len(base)] for i in range(S)]
        names = ['s%d' % i for i in range(S)]
        infos = []
        for i, sc in enumerate(seqs):
            infos += [dict(info, sequence_name=names[i]) for info in sc[1]]
        gt = ground_truth_from_infos(infos, names)
        res = track_sequences(torch.from_numpy(np.stack([sc[2] for sc in seqs])).cuda(), torch.from_numpy(np.stack([sc[3] for sc in seqs])),
                              torch.from_numpy(np.stack([sc[0]['poses'] for sc in seqs])), max_entries=1 << 20)
        te, all_e = timed(lambda: evaluate.evaluate_tracks(res, gt, CLASS_NAMES, CFG), a.reps)
        d, rec = evaluate.evaluate_tracks(res, gt, CLASS_NAMES, CFG, return_records=True)
        tab = evaluate.track_tables(res, gt, CLASS_NAMES)
        tm, all_m = timed(lambda: evaluate.tracking_metrics(**tab, breakdowns=CFG), a.reps)
        print(json.dumps({'S': S, 'frames': F, 'gt_per_frame': float(gt.counts.float().mean()),
                          'pred_per_frame': float(tab['pred_cnt'].float().mean()), 'evaluate_tracks_seconds': te,
                          'evaluate_tracks_frames_per_s': S * F / te, 'tracking_metrics_seconds': tm,
                          'tracking_metrics_frames_per_s': S * F / tm, 'vehicle_L2_MOTA': d['OBJECT_TYPE_TYPE_VEHICLE_LEVEL_2/MOTA'][0],
                          'mismatches_L2': int(rec[:4, 1, 0, 3].sum()), 'evaluate_tracks_all': all_e, 'tracking_metrics_all': all_m}),
              flush=True)
    if a.oracle_frames > 0:
        from oracle import track_eval_ref
        pred, pid, pc, gb, go, gty, gl, gc = (tab[k].cpu().numpy() for k in ('pred', 'pred_id', 'pred_cnt', 'gt_box', 'gt_obj',
                                                                               'gt_type', 'gt_level', 'gt_cnt'))
        n = min(a.oracle_frames, F)
        frames = [(pred[0, f, :pc[0, f]], pid[0, f, :pc[0, f]], gb[0, f, :gc[0, f]], go[0, f, :gc[0, f]], gty[0, f, :gc[0, f]],
                   gl[0, f, :gc[0, f]]) for f in range(n)]
        t0 = time.time()
        track_eval_ref.records([frames])
        dt = time.time() - t0
        print(json.dumps({'oracle_frames': n, 'oracle_seconds_per_frame': dt / n}), flush=True)


if __name__ == '__main__':
    main()

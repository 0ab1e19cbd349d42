"""Throughput of scoring tracks against ground truth on the device (detzero_b200.track.assign_track_target and tracklet_recall,
csrc/track_gt.cu): S in {1, 8, 64} full-scale sequences, each a 199-frame synthetic_sequence with 300 objects whose jittered
detections went through track_sequences (4 distinct sequences, repeated for S > 4).  Whole calls are timed with CUDA events after
a warm-up (assign_track_target includes its overflow check, tracklet_recall its one device-to-host copy and the host table).
Prints the card and its power limit, then one JSON line per S, and the numpy oracle's time on one sequence for scale."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detzero_b200 import synthetic                                                          # noqa: E402
from detzero_b200.track import assign_track_target, ground_truth_from_infos, track_sequences, tracklet_recall  # noqa: E402


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
    ap.add_argument('--no-oracle', action='store_true')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_track_gt needs a GPU'
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
        ta, all_a = timed(lambda: assign_track_target(res, gt), a.reps)
        tr, all_r = timed(lambda: tracklet_recall(res, gt), a.reps)
        m = assign_track_target(res, gt)
        print(json.dumps({'S': S, 'frames': F, 'objects_seq0': int(gt.n_obj[0]), 'tracks_seq0': int(res.n_tracks[0]),
                          'matches_seq0': len(m.matches(0)), 'assign_seconds': ta, 'assign_sequences_per_s': S / ta,
                          'recall_seconds': tr, 'recall_sequences_per_s': S / tr, 'assign_all': all_a, 'recall_all': all_r}),
              flush=True)
    if not a.no_oracle:
        from oracle import track_gt_ref
        tracks, _ = res.to_reference(names, gt.frame_ids)
        t0 = time.time()
        track_gt_ref.assign_track_target(seqs[0][1], tracks[names[0]], {'Vehicle': 0.3, 'Pedestrian': 0.1, 'Cyclist': 0.1})
        t1 = time.time()
        track_gt_ref.tracklet_recall([(seqs[0][1], tracks[names[0]])])
        t2 = time.time()
        print(json.dumps({'oracle_assign_seconds_per_sequence': t1 - t0, 'oracle_recall_seconds_per_sequence': t2 - t1}), flush=True)


if __name__ == '__main__':
    main()

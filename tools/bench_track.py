"""Throughput of the device tracker (detzero_b200.track.track_sequences): S in {1, 8, 64} sequences of 199 synthetic frames with
about 300 objects and 40 false positives per frame (synthetic.synthetic_detections; 8 distinct sequences, repeated for S = 64),
timed with CUDA events over whole calls (the call includes its host-side overflow check).  Prints the card and its power limit,
and checks every decision of sequence 0 against the numpy oracle (oracle.track_ref.check_device: keep flags, track ids, entry
frames, hit flags, classes, motion states; boxes to tolerance).  One JSON line per S."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detzero_b200 import synthetic                      # noqa: E402
from detzero_b200.track import tracker_cfg, track_sequences  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='1,8,64')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--no-oracle', action='store_true')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_track needs a GPU'
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print('card:', q.stdout.strip().splitlines()[0] if q.stdout else torch.cuda.get_device_name(0), flush=True)
    F = 199
    base = [synthetic.synthetic_detections(s, frames=F, objects=300, false_positives=40) for s in range(11, 19)]
    K = 500
    for S in [int(s) for s in a.sizes.split(',')]:
        seqs = [base[i % len(base)] for i in range(S)]
        boxes = torch.zeros((S, F, K, 9), dtype=torch.float32)
        for i, d in enumerate(seqs):
            boxes[i, :, :d['boxes'].shape[1]] = torch.from_numpy(d['boxes'])
        boxes = boxes.cuda()
        counts = torch.from_numpy(np.stack([d['counts'] for d in seqs])).cuda()
        poses = torch.from_numpy(np.stack([d['poses'] for d in seqs])).cuda()
        res = track_sequences(boxes, counts, poses)                   # warm-up
        torch.cuda.synchronize()
        times = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            res = track_sequences(boxes, counts, poses)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
        t = min(times)
        out = {'S': S, 'frames': F, 'seconds': t, 'all_seconds': times, 'sequences_per_s': S / t, 'frames_per_s': S * F / t,
               'tracks_seq0': int(res.n_tracks[0])}
        print(json.dumps(out), flush=True)
    if not a.no_oracle:
        from oracle import track_ref
        t0 = time.time()
        ref = track_ref.track_sequence(base[0]['boxes'], base[0]['counts'], base[0]['poses'], tracker_cfg())
        dt = time.time() - t0
        track_ref.check_device(res, 0, ref)                          # raises on any differing decision
        print(json.dumps({'oracle_seconds': dt, 'oracle_margin': ref['margin'].value, 'decisions_equal': True}), flush=True)


if __name__ == '__main__':
    main()

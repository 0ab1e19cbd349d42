"""The offboard chain of one sequence on the device: a 199-frame synthetic_sequence (180 K background points per frame plus the object
points, about 300 tracks of the three classes starting 6 to 150 m from the ego) -> jittered, shuffled detections with misses and far false positives
(synthetic.detections_from_sequence) -> track.track_sequences -> offboard.refine_sequence (PRM / GRM / CRM inputs and forwards in
chunks of 16 tracks per class, revert, combine_frames with the dropped detections).  Prints JSON lines with:
  * the card's name and power limit, read in the same run;
  * CUDA-event device time per stage of one timed run after a warm-up: track, each input kind, each forward, revert, combine (the
    combine_frames call with its two host reads), and their share of the chain;
  * sequences/s of the whole chain (track + refine_sequence, CUDA events around both, including the host stalls between kernels);
  * the combine_frames call on its own, best of --reps (memset, three kernels and its two host reads).

With --assign the tracks are also assigned to the sequence's ground truth (track.assign_track_target, outside the timed chain) and
every chunk is scored (refine.data.track_targets, refine.score): the stages 'targets' and 'score' then appear with their share.

    python tools/bench_offboard.py [--tracks 300] [--frames 199] [--background 180000] [--chunk 16] [--reps 5] [--assign]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from detzero_b200 import offboard, synthetic              # noqa: E402
from detzero_b200.refine import data as D                 # noqa: E402
from detzero_b200.track import assign_track_target, ground_truth_from_infos, track_sequences            # noqa: E402


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [v.strip() for v in q.split(',')]
    except Exception:
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--tracks', type=int, default=300)
    ap.add_argument('--frames', type=int, default=199)
    ap.add_argument('--background', type=int, default=180000)
    ap.add_argument('--chunk', type=int, default=16)
    ap.add_argument('--radius', type=float, default=150.0, help='objects start within this distance of the ego (m)')
    ap.add_argument('--mode', default='fp32', help='refiner COMPUTE_MODE')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--seed', type=int, default=1)
    ap.add_argument('--assign', action='store_true', help='score the refiners against the ground truth of the sequence')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_offboard needs a GPU'
    dev = torch.device('cuda:0')
    card, power = _card()
    print(json.dumps({'card': card, 'power_limit': power}), flush=True)
    t0 = time.time()
    s = synthetic.synthetic_sequence(a.seed, frames=a.frames, tracks=a.tracks, n_background=a.background, ego_step=0.0, max_speed=0.3,
                                     radius=a.radius)
    boxes, counts, _ = synthetic.detections_from_sequence(s, a.seed)
    gen_s = time.time() - t0
    frames, poses = torch.from_numpy(s['frames']).to(dev), torch.from_numpy(s['poses']).to(dev)
    boxes, counts, poses_h = torch.from_numpy(boxes).to(dev), torch.from_numpy(counts).to(dev), torch.from_numpy(s['poses']).to(dev)
    models = synthetic.refine_models(a.seed, mode=a.mode, device=dev)
    gt = ground_truth_from_infos(synthetic.synthetic_ground_truth(s, a.seed), ['seq'], device=dev) if a.assign else None

    def chain(timings=None):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        res = track_sequences(boxes, counts, poses_h, max_entries=1 << 20)
        ev[1].record()
        assign = assign_track_target(res, gt) if a.assign else None                 # not timed: it is not part of the chain
        ev[2].record()
        out = offboard.refine_sequence(frames, s['frame_offsets'], poses, res, models, chunk=a.chunk, seed=a.seed, timings=timings,
                                       assign=assign)
        ev[3].record()
        torch.cuda.synchronize()
        return res, out, ev[0].elapsed_time(ev[1]), ev[2].elapsed_time(ev[3])

    with torch.no_grad():
        chain()                                                                  # warm-up
        stages = {}
        res, out, track_ms, _ = chain(stages)                                    # stage times (one extra sync at the end)
        best = None
        for _ in range(2):
            _, _, t_ms, r_ms = chain()
            best = min(best or 1e30, t_ms + r_ms)
    stages = {'track': track_ms, **stages}
    total = sum(stages.values())
    n_tracks = int(res.n_tracks[0])
    print(json.dumps({'frames': a.frames, 'tracks': n_tracks, 'rows': int(out.count.sum()), 'chunk': a.chunk, 'mode': a.mode,
                      'stage_ms': {k: round(v, 3) for k, v in stages.items()},
                      'stage_share': {k: round(v / total, 4) for k, v in stages.items()},
                      'chain_ms': round(best, 2), 'sequences_per_s': round(1e3 / best, 3), 'tracks_per_s': round(n_tracks * 1e3 / best, 1),
                      'generate_s': round(gen_s, 1)}), flush=True)
    if a.assign:
        print(json.dumps({'scoring_share_of_chain': {k: round(stages[k] / total, 4) for k in ('targets', 'score')},
                          'recall': {c: {k: {n: v for n, v in r.items() if not isinstance(v, list)} for k, r in out.recall[c].items()}
                                     for c in out.recall}}), flush=True)

    t = out.tables
    drop = (res.boxes[0], res.counts[0], res.kept[0])
    args = [t[k] for k in ('prm_lidar', 'grm_pred', 'scores', 'frame_of_box', 'box_num', 'cls', 'track_id')]
    D.combine_frames(*args, a.frames, drop=drop)
    times = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        D.combine_frames(*args, a.frames, drop=drop)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    print(json.dumps({'combine_call_ms': round(min(times), 4), 'all_ms': [round(x, 4) for x in times],
                      'combine_share_of_chain': round(min(times) / best, 6)}), flush=True)


if __name__ == '__main__':
    main()

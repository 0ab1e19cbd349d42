"""Scoring the refiners against ground truth on the tools/bench_offboard.py sequence (199 frames, about 300 objects, tracked by
track.track_sequences and assigned by track.assign_track_target): CUDA-event time of refine.data.track_targets and of each record of
refine.score over all tracks of the sequence in one call, best of --reps after a warm-up, beside the host time of the numpy
restatement (oracle/refine_score_ref.py) on the same tracks, and the number of box pairs clipped per pass.  The refined boxes are
seeded perturbations of the ground truth (no refiner runs here).  Prints JSON lines, the card's name and power limit first.

About 30 K box pairs per pass are a few microseconds of arithmetic: what is measured is launch overhead, the small device-side
tensor operations around the kernels and the one device-to-host copy of each record.  No share of peak is claimed.

    python tools/bench_refine_score.py [--tracks 300] [--frames 199] [--reps 5] [--no-oracle]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_offboard import _card                           # noqa: E402
from detzero_b200 import synthetic                         # noqa: E402
from detzero_b200.refine import data as D                  # noqa: E402
from detzero_b200.refine import score as S                 # noqa: E402
from detzero_b200.track import assign_track_target, ground_truth_from_infos, track_sequences      # noqa: E402


def _best(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return round(min(times), 4), [round(t, 4) for t in times]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--tracks', type=int, default=300)
    ap.add_argument('--frames', type=int, default=199)
    ap.add_argument('--background', type=int, default=2000)
    ap.add_argument('--radius', type=float, default=150.0)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--seed', type=int, default=1)
    ap.add_argument('--no-oracle', action='store_true', help='skip the host restatement')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_refine_score needs a GPU'
    dev = torch.device('cuda:0')
    card, power = _card()
    print(json.dumps({'card': card, 'power_limit': power}), flush=True)
    s = synthetic.synthetic_sequence(a.seed, frames=a.frames, tracks=a.tracks, n_background=a.background, ego_step=0.0, max_speed=0.3,
                                     radius=a.radius)
    boxes, counts, _ = synthetic.detections_from_sequence(s, a.seed)
    infos = synthetic.synthetic_ground_truth(s, a.seed)
    res = track_sequences(torch.from_numpy(boxes)[None].to(dev), torch.from_numpy(counts)[None], torch.from_numpy(s['poses'])[None],
                          max_entries=1 << 20)
    gt = ground_truth_from_infos(infos, ['seq'], device=dev)
    assign = assign_track_target(res, gt)
    tb = res.track_batch()
    tg = D.track_targets(assign, tb)
    B, L = len(tb), tb.L
    g = torch.Generator(device=dev).manual_seed(a.seed)
    scored = tg.matched.bool() & tg.matched_tracklet.bool()[:, None]
    world = torch.where(scored[..., None], tg.gt_boxes, tb.boxes) + 0.05 * torch.randn((B, L, 7), generator=g, device=dev, dtype=torch.float64)
    grm = (tb.boxes[:, 0] * (1 + 0.05 * torch.randn((B, 7), generator=g, device=dev, dtype=torch.float64))).float()
    pred = torch.rand((B, L), generator=g, device=dev)
    th = [0.7]
    iou = S.refine_iou_labels(world, grm, tb, tg)
    n_scored, n_valid = int(scored.sum()), int(tb.box_num.sum())
    out = {'tracks': B, 'matched_tracks': int(tg.matched_tracklet.sum()), 'boxes': n_valid, 'reps': a.reps,
           'pairs_clipped': {'PRM': 2 * n_scored, 'GRM': 2 * n_scored, 'labels': n_valid, 'CRM': 0}}
    for name, fn in (('track_targets', lambda: D.track_targets(assign, tb)),
                     ('PRM', lambda: S.position_recall(world, tb, tg, th)),
                     ('GRM', lambda: S.geometry_recall(grm, tb, tg, th)),
                     ('labels', lambda: S.refine_iou_labels(world, grm, tb, tg)),
                     ('CRM', lambda: S.confidence_recall(tb.scores, pred, iou, tb, tg, th))):
        out[name + '_ms'], out[name + '_all_ms'] = _best(fn, a.reps)
    print(json.dumps(out), flush=True)
    if a.no_oracle:
        return
    from oracle import refine_score_ref as R
    from oracle import track_gt_ref
    tracks, _ = res.to_reference(['seq'], gt.frame_ids)
    t0 = time.time()
    assigned, _ = track_gt_ref.assign_track_target(infos, tracks['seq'], {'Vehicle': 0.3, 'Pedestrian': 0.1, 'Cyclist': 0.1})
    t_assign = time.time() - t0
    t0 = time.time()
    ti = R.attach_targets(assigned)
    ti = {t: ti[t] for t in tb.track_uid.cpu().tolist()}
    for i in ti.values():
        R.gt_pos_trajectory(i)
    host = {'targets_s': round(time.time() - t0, 3)}
    n = [len(i['boxes_global']) for i in ti.values()]
    w, gp = world.cpu().numpy(), grm.cpu().numpy()
    pw = [w[b, :k] for b, k in enumerate(n)]
    for name, fn in (('PRM', lambda: R.position_recall(ti, pw, th)), ('GRM', lambda: R.geometry_recall(ti, gp, th)),
                     ('labels', lambda: R.refine_iou_labels(ti, pw, gp))):
        t0 = time.time()
        r = fn()
        host[name + '_s'] = round(time.time() - t0, 3)
        if name == 'PRM':
            host['PRM_box_num'] = r[0]['Box num']
    host['assign_s (not part of the scoring)'] = round(t_assign, 1)
    print(json.dumps({'oracle_host': host, 'cpu': os.cpu_count(),
                      'device_PRM_box_num': S.position_recall(world, tb, tg, th)['Box num']}), flush=True)


if __name__ == '__main__':
    main()

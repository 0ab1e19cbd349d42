"""Refiner inputs on the device (detzero_b200/refine/data.py): a 199-frame synthetic sequence (180 K background points per frame plus
the object points), 256 tracks of 199 boxes (one per frame), built in chunks of 16 tracks.  Prints one JSON line:
  * device time per stage, from a torch.profiler run of its own: count (k_rd_crop<0>), select (k_rd_select), write (k_rd_crop<1>),
    fill + prep + scan (the rest of dz_refine_inputs), revert (k_rd_revert); and tracks/s for the PRM + GRM + CRM inputs (CUDA events,
    profiler off);
  * the count + write passes' algorithmic bytes -- encoded output rows x columns x 4, plus every point row of each box's frame read
    twice (count and write) x 24 bytes -- per second, as a share of 3.35 TB/s (H100 SXM data sheet).  A box re-reads the frame rows
    its neighbours in the same frame just read, so most of those reads are L2 hits and the share can exceed 1: it says how far the
    passes are from an HBM bound, not that HBM ran at that rate;
  * the whole chain -- crop + inputs -> PRM + GRM + CRM forward (production COMPUTE_MODE) -> revert -- in tracks/s;
  * the float64 numpy oracle (oracle/refine_data_ref.py) on the first --oracle-tracks tracks with every host thread, as a baseline;
  * the card's name and power limit, read in the same run.

    python tools/bench_refine_inputs.py [--tracks 256] [--frames 199] [--chunk 16] [--steps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from detzero_b200 import synthetic                          # noqa: E402
from detzero_b200.refine import data as D                   # noqa: E402

HBM = 3.35e12


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [v.strip() for v in q.split(',')]
    except Exception:
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def _oracle_track(args):
    from oracle import refine_data_ref as R
    s, b, seed = args
    one = {k: (v[b:b + 1] if k in ('boxes', 'frame_of_box', 'scores', 'box_num', 'cls', 'track_uid') else v) for k, v in s.items()}
    for kind in ('prm', 'grm', 'crm'):
        R.build_batch(kind, s['frames'], s['frame_offsets'], s['poses'], one, seed)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--tracks', type=int, default=256)
    ap.add_argument('--frames', type=int, default=199)
    ap.add_argument('--background', type=int, default=180000)
    ap.add_argument('--chunk', type=int, default=16)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--oracle-tracks', type=int, default=16)
    ap.add_argument('--seed', type=int, default=1)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_refine_inputs needs a GPU'
    dev = torch.device('cuda:0')
    card, power = _card()
    t0 = time.time()
    s = synthetic.synthetic_sequence(a.seed, frames=a.frames, tracks=a.tracks, n_background=a.background,
                                     lengths=[min(200, a.frames)] * a.tracks)
    gen_s = time.time() - t0
    frames = torch.from_numpy(s['frames']).to(dev)
    poses = torch.from_numpy(s['poses']).to(dev)
    off = s['frame_offsets']
    tb = D.TrackBatch(s['boxes'], s['frame_of_box'], s['scores'], s['box_num'], s['cls'], s['track_uid'], dev)
    chunks = [tb.select(slice(i, i + a.chunk)) for i in range(0, a.tracks, a.chunk)]

    def inputs(c):
        return (D.position_inputs(frames, off, poses, c, seed=a.seed), D.geometry_inputs(frames, off, poses, c, seed=a.seed),
                D.confidence_inputs(frames, off, poses, c, seed=a.seed))

    for c in chunks[:2]:
        inputs(c)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(a.steps):
        for c in chunks:
            inputs(c)
    ev[1].record()
    torch.cuda.synchronize()
    inputs_s = ev[0].elapsed_time(ev[1]) / 1e3 / a.steps

    # whole chain: crop + inputs -> PRM + GRM + CRM forward -> revert
    from detzero_b200.refine import ConfidencePointnet, GeometryTransformer, PositionTransformer
    from detzero_b200.synthetic import crm_cfg, grm_cfg, load_seeded, prm_cfg
    prm = PositionTransformer(prm_cfg(), 32, 32).eval(); load_seeded(prm, 1); prm = prm.to(dev)
    grm = GeometryTransformer(grm_cfg(), 11, 4).eval(); load_seeded(grm, 2); grm = grm.to(dev)
    crm = ConfidencePointnet(crm_cfg(), 32, 32).eval(); load_seeded(crm, 3); crm = crm.to(dev)

    def chain(c):
        p, g, q = inputs(c)
        bp = prm(p)['batch_box_preds']
        gp = grm(g)['batch_box_preds']
        crm(q)
        D.revert_position_boxes(bp, poses, c)
        D.revert_geometry_boxes(gp, poses, c)

    with torch.no_grad():
        for c in chunks[:2]:
            chain(c)
        torch.cuda.synchronize()
        ev[0].record()
        for c in chunks:
            chain(c)
        ev[1].record()
        torch.cuda.synchronize()
    chain_s = ev[0].elapsed_time(ev[1]) / 1e3

    # per-stage device time, profiler run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in chunks:
            p, g, q = inputs(c)
            D.revert_position_boxes(p['pos_trajectory'], poses, c)
            D.revert_geometry_boxes(g['geo_query_boxes'][:, 0], poses, c)
        torch.cuda.synchronize()
    stage = {'count': 0.0, 'select': 0.0, 'write': 0.0, 'prep_scan_fill': 0.0, 'revert': 0.0}
    for e in prof.key_averages():
        us = e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total
        n = e.key
        if 'k_rd_crop<0>' in n:
            stage['count'] += us
        elif 'k_rd_crop<1>' in n:
            stage['write'] += us
        elif 'k_rd_select' in n:
            stage['select'] += us
        elif 'k_rd_revert' in n:
            stage['revert'] += us
        elif 'k_rd_' in n:
            stage['prep_scan_fill'] += us
    stage = {k: v / 1e3 for k, v in stage.items()}                 # ms for all tracks, PRM + GRM + CRM

    # algorithmic bytes of the count + write passes (PRM + GRM + CRM)
    fsz = np.diff(off)
    rows_read = int(sum(fsz[s['frame_of_box'][b, :int(s['box_num'][b])]].sum() for b in range(a.tracks)))
    L = 200
    out_bytes = a.tracks * (L * (256 + 48) * 32 + L * 256 * 32 + 3 * 256 * 4 + 4096 * 11) * 4
    cw_bytes = out_bytes + 3 * 2 * rows_read * 24
    cw_s = (stage['count'] + stage['write']) / 1e3

    # oracle baseline with every host thread
    n_or = min(a.oracle_tracks, a.tracks)
    t0 = time.time()
    with ProcessPoolExecutor(max_workers=os.cpu_count()) as ex:
        list(ex.map(_oracle_track, [(s, b, a.seed) for b in range(n_or)]))
    oracle_s = time.time() - t0

    print(json.dumps({
        'metric': 'refine_inputs_tracks_per_s', 'value': round(a.tracks / inputs_s, 1),
        'card': card, 'power_limit': power,
        'tracks': a.tracks, 'boxes_per_track': int(s['box_num'][0]), 'frames': a.frames, 'points': int(off[-1]),
        'chunk': a.chunk, 'stage_ms_all_tracks': {k: round(v, 3) for k, v in stage.items()},
        'count_write_algorithmic_bw_over_hbm': round(cw_bytes / cw_s / HBM, 4) if cw_s > 0 else None,
        'count_write_bytes': cw_bytes,
        'chain_tracks_per_s': round(a.tracks / chain_s, 1),
        'oracle_cpu_tracks_per_s': round(n_or / oracle_s, 3), 'oracle_tracks': n_or, 'host_threads': os.cpu_count(),
        'sequence_gen_s': round(gen_s, 1)}))


if __name__ == '__main__':
    main()

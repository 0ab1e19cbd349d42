"""Is the neighbour gather what limits the bf16x2 sparse convs?  Times ``k_spconv_bf16`` on the real rulebooks of one
config-2 step (``bench.py``: 8 synthetic 180 K-point frames, VoxelBackBone8x) twice per layer:

  real     the layer's own neighbour table
  l2       a copy of that table in which every valid neighbour index i is replaced by i mod S (S = --rows, default 4096
           rows = 1 MB at Cin = 64): the same live rows, offsets, reduction blocks and MMAs, but every gathered row comes
           from a set that stays in L2
  one-row  a copy that keeps, per tile and offset, only the first valid neighbour: the same live blocks, MMAs and cp.async
           instructions, but nearly every copy is a zero-fill, so almost no bytes move from L2 to the SM

real / l2 says whether HBM traffic (the L2 misses of the gather) limits a layer; real / one-row says whether the bytes
moved into shared memory do.  If neither ratio is large, fetching fewer rows per tile cannot make the layer much faster.
Both the mask-grouped tile schedule and ``--no-schedule`` (rows in table order) are timed.  Only kernel times are read
(CUDA events around --reps launches, best of --rounds).

    python tools/probe_spconv_gather.py [--json OUT.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from detzero_b200 import _lib, ops
from detzero_b200 import synthetic as weights
from detzero_b200.det.centerpoint import build_network
from detzero_b200.spconv import pytorch as sp


def card():
    q = 'name,power.limit,clocks.max.sm'
    try:
        return subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=' + q, '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def capture_step(model, bd):
    """(args, kwargs) of every bf16-plane sparse-conv launch of one eager step, inputs kept alive"""
    calls, orig = [], ops.spconv_fwd

    def rec(*a, **k):
        out = orig(*a, **k)
        calls.append((a, dict(k)))
        return out
    ops.spconv_fwd = rec
    try:
        with torch.no_grad():
            model.forward_device(bd)
        torch.cuda.synchronize()
    finally:
        ops.spconv_fwd = orig
    return [(a, k) for a, k in calls if a[9] in _lib.PLANES]


def l2_tables(nbr, tab_tiles, K, S):
    """the same tables with every valid neighbour index i replaced by i mod S (the mask column and the row plane unchanged)"""
    t = nbr.clone()
    v = t[:, :K]
    t[:, :K] = torch.where(v >= 0, v % S, v)
    tt = None
    if tab_tiles is not None:
        tt = tab_tiles.clone()
        w = tt[:, :K, :]
        tt[:, :K, :] = torch.where(w >= 0, w % S, w)
    return t, tt


def one_row_tables(nbr, tab_tiles, K):
    """the same tables with, per tile and offset, only the first valid neighbour kept (the others -1): the tile's live offsets,
    reduction blocks, MMAs and cp.async instructions are unchanged, but almost every copy is a zero-fill that reads nothing"""
    def first_only(v, dim):
        ok = v >= 0
        return torch.where(ok & (ok.int().cumsum(dim) == 1), v, torch.full_like(v, -1))
    t = nbr.clone()
    T = t.shape[0] // 128                      # a ragged last capacity tile keeps its table
    t[:T * 128, :K] = first_only(t[:T * 128, :K].view(T, 128, K), 1).view(T * 128, K)
    tt = None
    if tab_tiles is not None:
        tt = tab_tiles.clone()
        tt[:, :K, :] = first_only(tt[:, :K, :], 2)
    return t, tt


def time_launch(a, k, nbr, tab_tiles, reps, rounds):
    a = list(a)
    a[1] = nbr
    k = dict(k)
    k['tab_tiles'] = tab_tiles
    k['out'] = torch.empty_like(ops.spconv_fwd(*a, **k))
    best = float('inf')
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.spconv_fwd(*a, **k)
        e1.record()
        torch.cuda.synchronize()
        best = min(best, 1000.0 * e0.elapsed_time(e1) / reps)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=4096, help='size of the L2-resident row set')
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'probe_spconv_gather.py needs a GPU'
    dev = torch.device('cuda', 0)
    sp_mode = os.environ.get('DZ_SP_MODE', weights.DEFAULT_SP_MODE)
    ds, batches = bench.build_inputs(8)
    model = build_network(bench.make_model_cfg('VoxelBackBone8x', 'tf32', sp_mode), 3, ds).eval()
    weights.load_seeded(model, 3)
    bench.tune_head_for_bench(model)
    model = model.to(dev)
    b = batches[0]
    pts = torch.from_numpy(b['points']).to(dev)
    bd = lambda: {'points': pts, 'points_per_frame': b['points_per_frame'], 'frame_id': b['frame_id'], 'batch_size': b['batch_size']}
    with torch.no_grad():
        for _ in range(3):                     # capacity hints settle
            try:
                model(bd())
            except RuntimeError as e:
                if 'overflow' not in str(e):
                    raise
    torch.cuda.synchronize()
    print('card: %s; sparse mode %s; L2 row set %d rows' % (card(), sp_mode, args.rows))
    rows = []
    for sched in (True, False):
        sp._SparseConv.SCHEDULE_TILES = sched
        calls = capture_step(model, bd())
        for i, (a, k) in enumerate(calls):
            K, cin, cout = k['kshape']
            subm = k.get('d_n_in') is None
            if not (subm and K == 27 and cin == cout and cin in (32, 64)):      # the 32- and 64-channel subm layers
                continue
            n_out = min(int(a[2].item()), a[3])
            nbr, tt = a[1], k.get('tab_tiles') if k.get('row_order') is not None else None
            l2n, l2t = l2_tables(nbr, tt, K, args.rows)
            pairs = int((nbr[:n_out, :K] >= 0).sum().item())
            us_real = time_launch(a, k, nbr, tt, args.reps, args.rounds)
            us_l2 = time_launch(a, k, l2n, l2t, args.reps, args.rounds)
            orn, ort = one_row_tables(nbr, tt, K)
            us_one_row = time_launch(a, k, orn, ort, args.reps, args.rounds)
            r = {'launch': i, 'schedule': sched, 'K': K, 'cin': cin, 'cout': cout, 'subm': subm, 'n_out': n_out, 'pairs': pairs,
                 'us_real': round(us_real, 1), 'us_l2': round(us_l2, 1), 'us_one_row': round(us_one_row, 1),
                 'speedup_l2': round(us_real / us_l2, 3), 'speedup_one_row': round(us_real / us_one_row, 3)}
            rows.append(r)
            print('%-11s launch %2d  K=%2d %3d->%-3d %s n_out=%7d pairs=%8d  real %7.1f us  l2 %7.1f us (x%.2f)  '
                  'one-row %7.1f us (x%.2f)' % ('schedule' if sched else 'no-schedule', i, K, cin, cout, 'subm' if subm else 'conv',
                                                n_out, pairs, us_real, us_l2, us_real / us_l2, us_one_row, us_real / us_one_row), flush=True)
    sp._SparseConv.SCHEDULE_TILES = True
    if args.json:
        with open(args.json, 'w') as f:
            json.dump({'card': card(), 'sp_mode': sp_mode, 'rows': args.rows, 'layers': rows}, f, indent=1)


if __name__ == '__main__':
    main()

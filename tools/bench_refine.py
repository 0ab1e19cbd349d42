#!/usr/bin/env python
"""Refiner throughput (BASELINE.json configs[3] shape family): GRM / PRM / CRM tracks per second on one GPU, next to the
same modules' CPU restatement timing is in BASELINE.md (reference PRM 1.12 s/track on 8 cores).

    python tools/bench_refine.py [--tracks 16] [--steps 5]

PRM: 200 boxes/track x 256 query pts (+48 memory pts) x 32 feats; GRM: 4096 memory pts x 11 + 3 x 256 x 4 queries;
CRM: 200 x 256 x 32.  Weights seeded.  Timed with CUDA events after warm-up; inputs resident on the device."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from oracle import refine_inputs as ri  # noqa: E402
from oracle import weights  # noqa: E402
from detzero_b200 import ops  # noqa: E402
from detzero_b200.refine import ConfidencePointnet, GeometryTransformer, PositionTransformer  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--tracks', type=int, default=16)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--mode', default='fp32')
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    out = {'tracks_per_step': a.tracks, 'steps': a.steps, 'mode': a.mode}
    for name, cls, cfg, dims, inputs in (('PRM', PositionTransformer, ri.prm_cfg(), (32, 32), ri.prm_inputs),
                                         ('GRM', GeometryTransformer, ri.grm_cfg(), (11, 4), ri.grm_inputs),
                                         ('CRM', ConfidencePointnet, ri.crm_cfg(), (32, 32), ri.crm_inputs)):
        cfg.COMPUTE_MODE = a.mode
        m = cls(cfg, *dims).eval()
        weights.load_seeded(m, 1)
        m = m.to(dev)
        d = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in inputs(5, B=a.tracks).items()}
        for _ in range(2):
            m(dict(d))
        torch.cuda.synchronize()
        ops.reset_launch_count()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(a.steps):
            m(dict(d))
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / a.steps
        out[name] = {'ms_per_step': ms, 'tracks_per_s': a.tracks / (ms / 1000.0), 'gpu_launches_per_step': ops.launch_count() // a.steps}
    print(json.dumps(out))


if __name__ == '__main__':
    main()

"""shared builders for the parity tests"""
import re

import numpy as np
import torch

from detzero_b200.config import AttrDict

SMALL_RANGE = [-9.6, -9.6, -2, 9.6, 9.6, 4]
VOXEL = [0.1, 0.1, 0.15]
WAYMO_RANGE = [-75.2, -75.2, -2, 75.2, 75.2, 4]


def config1_cloud(n=20000, seed=0, pc_range=WAYMO_RANGE, c=5):
    """SURVEY.md §8d config 1: uniform cloud + 2 % out-of-range + 5 % exact duplicates / on-lattice coordinates"""
    g = np.random.default_rng(seed)
    lo, hi = np.array(pc_range[:3], np.float32), np.array(pc_range[3:], np.float32)
    p = g.uniform(lo, hi, (n, 3)).astype(np.float32)
    n_out = n // 50
    p[:n_out] = p[:n_out] * 1.2 + np.array([3.0, -3.0, 5.0], np.float32)          # outside (some in z only)
    n_dup = n // 20
    src = g.integers(n_out, n, n_dup)
    dst = g.integers(n_out, n, n_dup)
    p[dst[: n_dup // 2]] = p[src[: n_dup // 2]]                                     # exact duplicates
    k = g.integers(-700, 700, (n_dup - n_dup // 2, 3)).astype(np.float32)
    p[dst[n_dup // 2:]] = (k * np.array(VOXEL, np.float32)).astype(np.float32)      # exactly on the lattice
    p[g.integers(0, n, 8), 0] = hi[0]                                               # x == upper bound exactly
    feats = np.concatenate([np.tanh(g.uniform(0, 2, (n, 1))), g.uniform(0, 1, (n, max(c - 4, 1)))], axis=1)
    return np.concatenate([p, feats.astype(np.float32)], axis=1)[:, :c].astype(np.float32)


def clustered_cloud(n, seed, pc_range=SMALL_RANGE, c=5):
    """points concentrated on a few surfaces so that voxels have neighbours (exercises the rulebook)"""
    g = np.random.default_rng(seed)
    lo, hi = np.array(pc_range[:3], np.float32), np.array(pc_range[3:], np.float32)
    xy = g.uniform(lo[:2], hi[:2], (n, 2))
    z = np.where(g.random(n) < 0.6, g.normal(0.0, 0.05, n), g.uniform(0, 2.5, n))
    wall = g.random(n) < 0.3
    xy[wall, 0] = np.round(xy[wall, 0] / 3.0) * 3.0 + g.normal(0, 0.03, wall.sum())
    p = np.concatenate([xy, z[:, None]], axis=1)
    f = np.concatenate([np.tanh(g.uniform(0, 2, (n, 1))), g.uniform(0, 1, (n, c - 4))], axis=1)
    return np.concatenate([p, f], axis=1).astype(np.float32)


from detzero_b200.synthetic import model_cfg, CLASS_NAMES    # noqa: E402,F401  (one definition, shared with bench.py)


def rel_err(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def assert_within(got, ref, bound, what):
    """|got - ref| <= bound element-wise; NaN exactly where ref is NaN.  Returns the largest err / bound; a failure reports it and
    where it occurs"""
    got = got.to(torch.float64)
    ref, bound = ref.to(got.device), bound.to(got.device)
    gn, rn = torch.isnan(got), torch.isnan(ref)
    if not torch.equal(gn, rn):
        i = np.unravel_index(int((gn != rn).to(torch.uint8).argmax()), tuple(got.shape))
        raise AssertionError('%s: NaN pattern differs from torch at %s (got %r, ref %r)' % (what, i, got[i].item(), ref[i].item()))
    err = torch.where(rn, torch.zeros_like(got), (got - ref).abs())
    bound = torch.where(rn, torch.zeros_like(bound), bound)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)      # bound == 0 and err > 0: inf
    ratio = torch.nan_to_num(ratio, nan=float('inf'))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if not worst <= 1.0:
        i = np.unravel_index(int(ratio.argmax()), tuple(got.shape))
        raise AssertionError('%s: largest err/bound %.3g at %s (err %.3g, bound %.3g, got %r, ref %r)'
                             % (what, worst, i, err[i].item(), bound[i].item(), got[i].item(), ref[i].item()))
    return worst


def assert_equal_signed(got, ref, what):
    """bit-level agreement up to NaN payloads: equal values and the same sign of zero"""
    got, ref = got.cpu(), ref.cpu().to(got.dtype)
    same = (got == ref) & (torch.signbit(got) == torch.signbit(ref))
    if not bool(same.all()):
        i = np.unravel_index(int((~same).to(torch.uint8).argmax()), tuple(got.shape))
        raise AssertionError('%s: first difference at %s (got %r, torch %r)' % (what, i, got[i].item(), ref[i].item()))


def _conv2d_kernel_names(prof):
    seen = set()
    for e in prof.key_averages():
        m = re.search(r'(k_conv2d_tf32_halo_n256|k_conv2d_tf32|k_conv2d_f32)<([^>]*)>', e.key)
        if m:
            args = [re.sub(r'\((?:int|bool)\)', '', a).strip() for a in m.group(2).split(',')]
            if m.group(1) == 'k_conv2d_tf32':
                args[1] = {'0': 'false', '1': 'true'}.get(args[1], args[1])
            seen.add('%s<%s>' % (m.group(1), ', '.join(args)))
    return seen


def conv2d_kernels(run, tries=3):
    """(run(), the dense conv2d kernels it launched as 'name<args>' with the demangler's (int) / (bool) casts removed), from
    torch.profiler.  A profiler session now and then records none of its kernels; run (idempotent) is then profiled again, so a
    lost record is not taken for a wrong kernel, while a wrong kernel still shows as one"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = run()
            torch.cuda.synchronize()
        seen = _conv2d_kernel_names(prof)
        if seen:
            break
    return out, seen

"""The gather probe (tools/probe_spconv_gather.py) compares a layer's launch with launches on rewritten neighbour tables.  The
comparison only means something if the rewrites keep every tile's live offsets, reduction blocks and MMAs: checked here on
the CPU, for both the row-major table and the tile-major scheduled table."""
import importlib.util
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location('probe_spconv_gather', os.path.join(ROOT, 'tools', 'probe_spconv_gather.py'))
probe = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(probe)

K = 27


def _tables(seed, rows=300, tiles=3):
    g = torch.Generator().manual_seed(seed)
    tab = torch.randint(0, 200000, (rows, 32), generator=g, dtype=torch.int32)
    tab[:, :K][torch.rand((rows, K), generator=g) < 0.6] = -1
    tab[:, 27] = ((tab[:, :K] >= 0).long() << torch.arange(K)).sum(1).int()
    tt = torch.randint(0, 200000, (tiles, K + 1, 128), generator=g, dtype=torch.int32)
    tt[:, :K][torch.rand((tiles, K, 128), generator=g) < 0.6] = -1
    tt[:, :K, 0:8] = -1                                       # an offset with no live row in part of a tile
    tt[1, 5] = -1                                             # an offset dead in a whole tile
    return tab, tt


def test_l2_tables_keep_the_live_pattern():
    tab, tt = _tables(0)
    S = 4096
    t2, tt2 = probe.l2_tables(tab, tt, K, S)
    assert torch.equal(t2[:, K:], tab[:, K:]) and torch.equal(tt2[:, K], tt[:, K])
    assert torch.equal(t2[:, :K] >= 0, tab[:, :K] >= 0) and torch.equal(tt2[:, :K] >= 0, tt[:, :K] >= 0)
    assert int(t2[:, :K].max()) < S and int(tt2[:, :K].max()) < S
    valid = tab[:, :K] >= 0
    assert torch.equal(t2[:, :K][valid], tab[:, :K][valid] % S)


def test_one_row_tables_keep_one_row_per_live_tile_offset():
    tab, tt = _tables(1)
    t2, tt2 = probe.one_row_tables(tab, tt, K)
    assert torch.equal(t2[:, K:], tab[:, K:]) and torch.equal(tt2[:, K], tt[:, K])
    T = tab.shape[0] // 128
    assert torch.equal(t2[T * 128:], tab[T * 128:])           # the ragged capacity tail is left as it is
    for new, old, dim in ((t2[:T * 128, :K].view(T, 128, K), tab[:T * 128, :K].view(T, 128, K), 1), (tt2[:, :K], tt[:, :K], 2)):
        live_old, live_new = (old >= 0).any(dim), (new >= 0).sum(dim)
        assert torch.equal(live_new, live_old.int())          # same live (tile, offset) pairs, one row each
        kept = new >= 0
        assert torch.equal(new[kept], old[kept])              # the kept row is the original one ...
        first = (old >= 0).int().cumsum(dim) == 1
        assert bool((first & (old >= 0))[kept].all())         # ... and the first valid one of its (tile, offset)

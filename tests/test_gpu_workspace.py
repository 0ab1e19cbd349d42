"""Every C-ABI entry point that takes a scratch workspace, called through ctypes at the size its *_ws_bytes reports: at one realistic
and one edge shape each, a call given exactly that many bytes gives the same outputs as one given a generous workspace and writes
nothing past them (a sentinel tail follows the workspace), and a call given one byte less returns DZ_ERR_WORKSPACE before it
enqueues anything, so its outputs stay as they were."""
import ctypes

import numpy as np
import pytest
import torch

from detzero_b200 import _lib, ops, synthetic
from detzero_b200.refine import data as D
from tests import util

pytestmark = pytest.mark.gpu

DZ_ERR_WORKSPACE = -3
FILL, SENTINEL, TAIL = 0xA5, 0x5A, 4096
L = _lib.lib
P = ops._p


def _bits(t):
    return t.detach().reshape(-1).view(torch.uint8).clone()


def _blank(*shape, dtype=torch.float32):
    """an output that starts as a byte pattern no kernel writes on its own"""
    t = torch.empty(*shape, dtype=dtype, device='cuda')
    t.view(torch.uint8).fill_(0x3C)
    return t


def _run(setup, ws, nbytes):
    call, outs = setup()
    before = [_bits(o) for o in outs]
    rc = call(ws, nbytes)
    torch.cuda.synchronize()
    return rc, outs, before


def check_workspace(nbytes, setup, same=None):
    """setup() -> (call(ws, ws_bytes) -> rc, outputs), on fresh inputs each time; same(got, want) compares the outputs of two
    successful calls (default: bit for bit)"""
    assert nbytes >= 1
    big = torch.full((nbytes + (1 << 20),), FILL, dtype=torch.uint8, device='cuda')
    rc, want, _ = _run(setup, big, big.numel())
    assert rc == 0, L().dz_last_error_string()
    buf = torch.full((nbytes + TAIL,), FILL, dtype=torch.uint8, device='cuda')
    buf[nbytes:] = SENTINEL
    rc, got, _ = _run(setup, buf, nbytes)
    assert rc == 0, L().dz_last_error_string()
    if same is None:
        for i, (g, w) in enumerate(zip(got, want)):
            assert torch.equal(_bits(g), _bits(w)), i
    else:
        same(got, want)
    assert bool((buf[nbytes:] == SENTINEL).all())
    rc, after, before = _run(setup, buf, nbytes - 1)
    assert rc == DZ_ERR_WORKSPACE
    for i, (a, b) in enumerate(zip(after, before)):
        assert torch.equal(_bits(a), b), i


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


# ---- grid index scan, voxelization ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('words', [2 * 41 * 192 * 192 // 32, 1])
def test_grid_index_scan(cuda, words):
    bitmap = torch.randint(-2 ** 31, 2 ** 31 - 1, (words,), generator=_gen(1), dtype=torch.int32, device=cuda)

    def setup():
        prefix, total = _blank(words, dtype=torch.int32), _blank(1, dtype=torch.int32)
        return (lambda ws, nb: L().dz_grid_index_scan(P(bitmap), P(prefix), words, None, P(total), P(ws), nb, ops._stream()),
                [prefix, total])
    check_workspace(L().dz_scan_ws_bytes(words), setup)


GRID_ZYX, DHW, MAX_PTS = [40, 192, 192], [41, 192, 192], 5


def _cloud(n, seed):
    return torch.from_numpy(util.clustered_cloud(n, seed) if n else np.zeros((0, 5), np.float32)).float().contiguous().cuda()


def _vox_outputs(cap, B, n_tot):
    counters = torch.zeros(3, dtype=torch.int32, device='cuda')
    index = ops.GridIndex(B, DHW, 'cuda', with_perm_cap=n_tot + 1)
    for t in (index.prefix, index.perm):                # rows past the occupied cells are never written
        t.view(torch.uint8).fill_(0x3C)
    return [_blank(cap, MAX_PTS, 5), _blank(cap, 4, dtype=torch.int32), _blank(cap, dtype=torch.int32), _blank(cap, 5), counters,
            index.bitmap, index.prefix, index.perm]


@pytest.mark.parametrize('n,max_voxels', [(20000, 16000), (1, 16000), (0, 16000)])
def test_voxelize_hard(cuda, n, max_voxels):
    pts = _cloud(n, 2)
    cap = max(min(n, max_voxels), 1)

    def setup():
        o = _vox_outputs(cap, 1, n)
        return (lambda ws, nb: L().dz_voxelize_hard(P(pts) if n else None, n, 5, 0, 5, _lib.farr(util.SMALL_RANGE),
                                                   _lib.farr(util.VOXEL), _lib.iarr(GRID_ZYX), MAX_PTS, max_voxels, 0,
                                                   *[P(t) for t in o[:4]], cap, P(o[4]), 1, *DHW, *[P(t) for t in o[5:]],
                                                   P(ws), nb, ops._stream())), o
    check_workspace(L().dz_voxelize_hard_ws_bytes(n, MAX_PTS, max_voxels, *DHW), setup)


@pytest.mark.parametrize('ns', [[20000, 0, 1, 15000, 20000, 7, 18000, 3000], [5000]])
def test_voxelize_hard_batch(cuda, ns):
    """frames of unequal size: each is carved with its own count inside a slice sized for the largest"""
    clouds = [_cloud(n, 10 + b) for b, n in enumerate(ns)]
    B, max_voxels = len(ns), 16000
    cap = sum(min(n, max_voxels) for n in ns)
    ptrs = (ctypes.c_void_p * B)(*[c.data_ptr() if c.shape[0] else None for c in clouds])
    n_host = (ctypes.c_int * B)(*ns)

    def setup():
        o = _vox_outputs(cap, B, sum(ns))
        return (lambda ws, nb: L().dz_voxelize_hard_batch(ptrs, n_host, B, 5, 0, 5, _lib.farr(util.SMALL_RANGE), _lib.farr(util.VOXEL),
                                                         _lib.iarr(GRID_ZYX), MAX_PTS, max_voxels, *[P(t) for t in o[:4]], cap,
                                                         P(o[4]), *DHW, *[P(t) for t in o[5:]], P(ws), nb, ops._stream())), o
    check_workspace(L().dz_voxelize_hard_batch_ws_bytes(max(ns), B, MAX_PTS, max_voxels, *DHW), setup)


@pytest.mark.parametrize('n,B', [(60000, 2), (1, 1), (0, 1)])
def test_voxelize_dynamic(cuda, n, B):
    pts = np.concatenate([np.pad(util.clustered_cloud(n // B, 20 + b, c=4), ((0, 0), (1, 0)), constant_values=b) for b in range(B)])
    pts = torch.from_numpy(pts).cuda() if n else torch.zeros((1, 5), device=cuda)
    cap, grid = max(n, 1), [192, 192, 40]

    def setup():
        o = [_blank(cap, 4), _blank(cap, 4, dtype=torch.int32), _blank(1, dtype=torch.int32)]
        return (lambda ws, nb: L().dz_voxelize_dynamic_mean(P(pts), n, 4, B, _lib.farr(util.SMALL_RANGE), _lib.farr(util.VOXEL),
                                                           _lib.iarr(grid), P(o[0]), P(o[1]), cap, P(o[2]), P(ws), nb,
                                                           ops._stream())), o
    check_workspace(L().dz_voxelize_dynamic_ws_bytes(n, cap, B, *grid), setup)


# ---- rulebook tile schedule ----------------------------------------------------------------------------------------------------
def _schedule_valid(order, tab_tiles, tab, n, cap, K):
    """the schedule is built with atomics, so two runs may order rows of one digest (and tiles of one weight) differently; what
    both must satisfy: order[:n] is a permutation of the rows, the tile order a permutation of the tiles with non-increasing live
    offsets, each tile mask the OR of its rows' masks, and the tile-major table the table's rows in schedule order"""
    tiles = (cap + 127) // 128
    tab = tab.cpu()
    o = order.long().cpu()
    assert torch.equal(o[:n].sort().values, torch.arange(n))
    tile_order, tile_mask = o[cap:cap + tiles], order[cap + tiles:].cpu()
    assert torch.equal(tile_order.sort().values, torch.arange(tiles))
    rows = torch.full((tiles * 128,), -1, dtype=torch.long)
    rows[:n] = o[:n]
    masks = torch.where(rows >= 0, tab[rows.clamp(min=0), 27], 0).reshape(tiles, 128)
    ored = torch.zeros(tiles, dtype=torch.int32)
    for j in range(128):
        ored |= masks[:, j]
    assert torch.equal(ored, tile_mask)
    live = torch.tensor([bin(int(m) & 0xFFFFFFFF).count('1') for m in tile_mask[tile_order]])
    assert bool((live[:-1] >= live[1:]).all())
    tt = tab_tiles.cpu()[:(n + 127) // 128]
    want = torch.where(rows[:, None] >= 0, tab[rows.clamp(min=0), :K], -1).reshape(tiles, 128, K)[:(n + 127) // 128]
    assert torch.equal(tt[:, :K].permute(0, 2, 1), want)
    assert torch.equal(tt[:, K].reshape(-1), rows[:tt.shape[0] * 128].int())


@pytest.mark.parametrize('n,cap', [(40000, 40960), (777, 1000)])
def test_rulebook_schedule(cuda, n, cap):
    """the rulebook kernel fills the scratch (histogram, tile masks and tickets zeroed first) and the schedule reads it; cap 1000
    is not a multiple of the 128-row tile"""
    g = np.random.default_rng(5)
    cells = np.sort(g.choice(41 * 192 * 192, n, replace=False))
    coords = np.zeros((cap, 4), np.int32)
    coords[:n, 1], coords[:n, 2], coords[:n, 3] = cells // (192 * 192), cells // 192 % 192, cells % 192
    coords = torch.from_numpy(coords).cuda()
    d_n = torch.tensor([n], dtype=torch.int32, device=cuda)
    gi = ops.grid_index_from_coords(coords, d_n, cap, 1, DHW)
    K = 27
    tiles = (cap + 127) // 128
    tab = ops.rulebook_subm(coords, d_n, cap, gi, [3, 3, 3], layout='row')

    def setup():
        o = [_blank(cap + 2 * tiles, dtype=torch.int32), _blank(tiles, K + 1, 128, dtype=torch.int32)]

        def call(ws, nb):
            rc = L().dz_rulebook_subm(P(coords), P(d_n), cap, 1, *DHW, _lib.iarr([3, 3, 3]), P(gi.bitmap), P(gi.prefix), P(gi.perm),
                                      None, P(tab), P(ws), ops._stream())
            assert rc == 0
            return L().dz_rulebook_schedule(P(tab), cap, P(d_n), P(o[0]), P(ws), nb, K, P(o[1]), ops._stream())
        return call, o

    def same(got, want):
        for order, tab_tiles in (got, want):
            _schedule_valid(order, tab_tiles, tab, n, cap, K)
    check_workspace(L().dz_rulebook_schedule_ws_bytes(cap), setup, same)


# ---- CenterHead decode, NMS --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,H,W,C,K,thresh', [(2, 188, 188, 3, 500, 0.1), (1, 4, 4, 1, 1, -1.0)])
def test_centerhead_decode(cuda, B, H, W, C, K, thresh):
    head = torch.randn(B, H, W, 9 + C, generator=_gen(3), device=cuda)

    def setup():
        o = [_blank(B, K, 7), _blank(B, K), _blank(B, K, dtype=torch.int32), _blank(B, dtype=torch.int32)]
        return (lambda ws, nb: L().dz_centerhead_decode(P(head), B, H, W, 9 + C, 0, 2, 3, 6, 8, 9, C, K,
                                                       _lib.farr([-75.2, -75.2, -2, 75.2, 75.2, 4]), _lib.farr([0.1, 0.1, 0.15]), 8,
                                                       _lib.farr([-80, -80, -10, 80, 80, 10]), thresh, 1, *[P(t) for t in o], P(ws), nb,
                                                       ops._stream())), o
    check_workspace(L().dz_centerhead_decode_ws_bytes(B, H, W, C, K), setup)


@pytest.mark.parametrize('ns,cap', [([900, 1024], 1024), ([1], 1)])
def test_nms_bev(cuda, ns, cap):
    B, post_max = len(ns), 83
    g = np.random.default_rng(4)
    boxes = np.concatenate([g.uniform(-40, 40, (B, cap, 3)), g.uniform(1, 5, (B, cap, 3)), g.uniform(-np.pi, np.pi, (B, cap, 1))], 2)
    boxes = torch.from_numpy(boxes.astype(np.float32)).cuda()
    scores = torch.rand(B, cap, generator=_gen(4), device=cuda)
    labels = torch.randint(1, 4, (B, cap), generator=_gen(5), device=cuda, dtype=torch.int32)
    d_n = torch.tensor(ns, dtype=torch.int32, device=cuda)

    def setup():
        o = [_blank(B, post_max, 9), _blank(B, dtype=torch.int32)]
        return (lambda ws, nb: L().dz_nms_bev(P(boxes), P(scores), P(labels), P(d_n), B, cap, ctypes.c_float(0.1), post_max, 1,
                                             P(o[0]), P(o[1]), P(ws), nb, ops._stream())), o
    check_workspace(L().dz_nms_bev_ws_bytes(B, cap), setup)


# ---- point preparation, crops --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [180000, 1])
def test_prepare_points(cuda, n):
    raw = torch.randn(n, 6, generator=_gen(6), device=cuda) * 30
    t12 = (ctypes.c_double * 12)(*[1, 0, 0, 0.5, 0, 1, 0, -2, 0, 0, 1, 0.25])
    cap = n + 5

    def setup():
        o = [_blank(cap, 6), torch.zeros(1, dtype=torch.int32, device=cuda)]
        return (lambda ws, nb: L().dz_prepare_points(P(raw), n, t12, 0.0, 0, 1, P(o[0]), cap, P(o[1]), P(ws), nb, ops._stream())), o
    check_workspace(L().dz_prepare_points_ws_bytes(n), setup)


@pytest.mark.parametrize('M,T', [(100000, 64), (1, 1), (0, 1)])
def test_crop_points_in_boxes(cuda, M, T):
    pts = (torch.rand(max(M, 1), 4, generator=_gen(7), device=cuda) - 0.5) * 40
    g = np.random.default_rng(7)
    boxes = np.concatenate([g.uniform(-15, 15, (T, 3)), g.uniform(2, 8, (T, 3)), g.uniform(-np.pi, np.pi, (T, 1))], 1)
    boxes = torch.from_numpy(boxes.astype(np.float32)).cuda()
    cap = 512

    def setup():
        o = [_blank(T, cap, dtype=torch.int32), _blank(T, dtype=torch.int32)]
        return (lambda ws, nb: L().dz_crop_points_in_boxes(P(pts), M, 4, P(boxes), T, 7, P(o[0]), cap, P(o[1]), P(ws), nb,
                                                          ops._stream())), o
    check_workspace(L().dz_crop_points_ws_bytes(M, T), setup)


# ---- refiner inputs, combine, WBF ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind,tracks,lengths', [(D.PRM, 10, [24, 1, 2, 17, 24, 5, 9, 24, 3, 12]), (D.CRM, 1, [1]), (D.GRM, 1, [1])])
def test_refine_inputs(cuda, kind, tracks, lengths):
    s = synthetic.synthetic_sequence(3, frames=24, tracks=tracks, n_background=20000, lengths=lengths)
    tb = D.TrackBatch(s['boxes'], s['frame_of_box'], s['scores'], s['box_num'], s['cls'], s['track_uid'], cuda)
    frames = torch.from_numpy(s['frames']).to(cuda)
    off, F, max_pts, poses = D._frames_args(frames, s['frame_offsets'], torch.from_numpy(s['poses']))
    B, Lb = len(tb), tb.L
    kq, km, nq = (256, 48, 1) if kind == D.PRM else (256, 0, 1) if kind == D.CRM else (256, 4096, 3)
    q_out = min(nq, tb.max_box_num) if kind == D.GRM else 0
    C = 4 if kind == D.GRM else 32

    def setup():
        if kind == D.GRM:
            o = [_blank(B, q_out, kq, 4), _blank(B, km, 11), _blank(B, Lb, 7), _blank(B, q_out, 7), None, _blank(B, dtype=torch.int32)]
            nsel = nq * kq + km
        else:
            o = [_blank(B, Lb, kq, C), _blank(B, Lb, km, C) if kind == D.PRM else None, _blank(B, Lb, 7) if kind == D.PRM else None,
                 _blank(B, Lb), _blank(B, 7) if kind == D.PRM else None, None]
            nsel = Lb * (kq + km)
        o += [_blank(B, Lb, dtype=torch.int32), _blank(B, nsel, dtype=torch.int32)]
        call = (lambda ws, nb: L().dz_refine_inputs(kind, P(frames), frames.stride(0), P(off), F, max_pts, P(poses), P(tb.boxes),
                                                    P(tb.frame_of_box), P(tb.scores), P(tb.box_num), P(tb.cls), P(tb.track_uid),
                                                    B, Lb, kq, km, nq, q_out, 0, 1.1, 0, 1, 7, *[P(t) for t in o], P(ws), nb,
                                                    ops._stream()))
        return call, [t for t in o if t is not None]
    check_workspace(L().dz_refine_inputs_ws_bytes(kind, B, Lb, max_pts, kq, km, nq), setup)


@pytest.mark.parametrize('B,F,Lb,K', [(300, 199, 200, 500), (1, 1, 1, 1)])
def test_combine_frames(cuda, B, F, Lb, K):
    g = np.random.default_rng(8)
    n = g.integers(1, min(F, Lb) + 1, B).astype(np.int32)
    fob = np.zeros((B, Lb), np.int32)
    for b in range(B):
        fob[b, :n[b]] = np.arange(n[b]) + g.integers(0, F - n[b] + 1)
    dev = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(device=cuda, dtype=dt)  # noqa: E731
    prm = dev(np.concatenate([g.uniform(-80, 80, (B, Lb, 3)), g.uniform(0.5, 5, (B, Lb, 3)), g.uniform(-7, 7, (B, Lb, 1))], 2),
              torch.float64)
    grm, sc = dev(g.normal(0, 3, (B, 7)), torch.float32), dev(g.uniform(0, 1, (B, Lb)), torch.float32)
    fob, bn, cls = dev(fob, torch.int32), dev(n, torch.int32), dev(g.integers(1, 4, B), torch.int32)
    tid = dev(g.permutation(100000)[:B], torch.int32)
    det = np.zeros((F, K, 9), np.float32)
    det[..., :7], det[..., 7], det[..., 8] = g.uniform(-20, 20, (F, K, 7)), g.uniform(0, 1, (F, K)), g.integers(1, 4, (F, K))
    det, cnt, kept = dev(det, torch.float32), dev(g.integers(0, K + 1, F), torch.int32), dev(g.random((F, K)) < 0.3, torch.uint8)
    R = 1024

    def setup():
        o = [_blank(F, R, 9), _blank(F, R, dtype=torch.int32), _blank(F, dtype=torch.int32), torch.zeros(1, dtype=torch.int32, device=cuda)]
        return (lambda ws, nb: L().dz_combine_frames(P(prm), P(grm), P(sc), P(fob), P(bn), P(cls), P(tid), B, Lb, P(det), P(cnt),
                                                    P(kept), K, F, R, *[P(t) for t in o], P(ws), nb, ops._stream())), o
    check_workspace(L().dz_combine_frames_ws_bytes(B, Lb, F), setup)


@pytest.mark.parametrize('B,V,K', [(4, 4, 500), (1, 1, 1)])
def test_wbf_3d(cuda, B, V, K):
    g = np.random.default_rng(9)
    obj = np.concatenate([g.uniform(-30, 30, (60, 3)), g.uniform(1, 4, (60, 3)), g.uniform(-np.pi, np.pi, (60, 1))], 1)
    pick = g.integers(0, 60, (B * V, K))
    rows = np.zeros((B * V, K, 9), np.float32)
    rows[..., :7] = obj[pick] + g.normal(0, 0.1, (B * V, K, 7))
    rows[..., 7], rows[..., 8] = g.uniform(0, 1, (B * V, K)), pick % 3 + 1
    rows = torch.from_numpy(rows).cuda()
    counts = torch.from_numpy(g.integers(0, K + 1, B * V).astype(np.int32)).cuda()
    iou, skip = [0.55, 0.5, 0.5], [0.0, 0.0, 0.0]

    def setup():
        o = [_blank(B, V * K, 9), _blank(B, dtype=torch.int32)]
        return (lambda ws, nb: L().dz_wbf_3d(P(rows), P(counts), B, V, K, _lib.darr(iou), _lib.darr(skip), 3, P(o[0]), P(o[1]),
                                            P(ws), nb, ops._stream())), o
    check_workspace(L().dz_wbf_3d_ws_bytes(B, V, K, 3), setup)


# ---- training passes ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('crops,Pc,c0', [(256, 256, 32), (1, 64, 8)])
def test_crm_point_pass(cuda, crops, Pc, c0):
    """pass 5, whose slab partials are zeroed in the workspace before the kernel accumulates into them"""
    gen = _gen(10)
    x = torch.randn(crops * Pc, c0, generator=gen, device=cuda)
    W = [torch.randn(n, k, generator=gen, device=cuda) / k ** 0.5 for n, k in ((128, c0), (128, 128), (256, 128), (256, 128))]
    wf = [w.t().contiguous() for w in W]
    tab = torch.rand(4, 6, 256, generator=gen, device=cuda) + 0.5
    shift4 = torch.randn(crops, 256, generator=gen, device=cuda)
    sel = torch.randint(0, Pc, (2, crops, 256), generator=gen, device=cuda, dtype=torch.int32)
    dsel = torch.randn(2, crops, 256, generator=gen, device=cuda)

    def setup():
        o = [_blank(512, dtype=torch.float64), _blank(2 * 256 * 128, dtype=torch.float64)]
        return (lambda ws, nb: L().dz_crm_point_pass(5, _lib.DZ_F32, P(x), crops, Pc, c0, *[P(w) for w in wf], P(W[1]), P(W[2]), P(W[3]),
                                                    P(tab), P(shift4), P(sel), P(dsel), None, None, None, P(o[0]), P(o[1]), P(ws), nb,
                                                    ops._stream())), o
    check_workspace(L().dz_crm_point_ws_bytes(crops), setup)


@pytest.mark.parametrize('R,gsize,N,K', [(4096, 256, 256, 128), (64, 64, 128, 11)])
def test_pm_wgrad(cuda, R, gsize, N, K):
    gen = _gen(11)
    dh, z, x = (torch.randn(R, c, generator=gen, device=cuda) for c in (N, N, K))
    tab = torch.rand(6, N, generator=gen, device=cuda) + 0.5

    def setup():
        o = [_blank(N, K, dtype=torch.float64)]
        return (lambda ws, nb: L().dz_pm_wgrad(_lib.DZ_F32, R, gsize, N, P(dh), None, None, P(z), P(tab), P(x), K, None, P(o[0]),
                                              P(ws), nb, ops._stream())), o
    check_workspace(L().dz_pm_wgrad_ws_bytes(R, N, K), setup)

"""Detection post-processing kernels element by element against float64 references, at their tie, boundary and capacity edges:
the rotated-BEV box geometry of csrc/boxgeom.cuh through every entry point that exposes it, the device NMS (k_nms_mask /
k_nms_scan) and the CenterHead top-K + decode (k_score_prefilter / k_topk_from_candidates / k_topk_class / k_topk_merge_decode).

Tolerances are derived from float32's unit roundoff U = 2^-24 and the CUDA maths library's documented error bounds (expf 2 ulp,
atan2f 3 ulp, cosf / sinf 2 ulp); one ulp of a value v is at most 2U|v|."""
import ctypes

import numpy as np
import pytest
import torch

from detzero_b200 import _lib, ops
from detzero_b200.refine.score import boxes_iou3d_aligned
from detzero_b200.track import IOU_2D, IOU_3D, IOU_BEV, OVERLAP_BEV, boxes_pairwise, points_in_boxes_gpu_v2
from tests import boxgeom_ref as gr

pytestmark = pytest.mark.gpu

U = gr.U


# ---- box geometry ---------------------------------------------------------------------------------------------------------
def _rows(x, cuda, ld=9):
    """float32 (n, 7) -> CUDA rows with a row stride of `ld` (the tracker reads boxes out of (F, 500, 9) rows)"""
    t = torch.full((x.shape[0], ld), 7.5, dtype=torch.float32, device=cuda)
    t[:, :7] = torch.from_numpy(x)
    return t[:, :7]


def _ratio_bound(o, d_o, S, floor):
    """bound on |fl(o' / max(S - o', floor)) - o / max(S - o, floor)| for |o' - o| <= d_o: d_o times the derivative, S / (S - o)^2
    (1 / floor where the guard holds), plus 4 roundings (the areas or volumes, the subtraction, the division) of the ratio"""
    un = np.maximum(S - o - d_o, floor)
    return d_o * np.maximum(S, un) / un ** 2 + 4 * U * o / un


def _ratio(o, S, floor):
    return o / np.maximum(S - o, floor)


@pytest.mark.parametrize('family', gr.FAMILIES)
def test_box_geometry_vs_float64(cuda, family):
    """BEV overlap, BEV IoU (dz_boxes_iou_bev and dz_boxes_pairwise), 3-D IoU (pairwise and aligned) and the axis-aligned 2-D
    IoU per pair: equal to the float64 restatement within the derived bound wherever every discrete test of the algorithm is
    decided by more than its rounding bound, inside the [exact, exact grown by the 1e-2 margin] envelope everywhere, exactly 0
    beyond the far_pair radius"""
    n = 256
    a, b = gr.pair_family(family, n)
    ta, tb = _rows(a, cuda), _rows(b, cuda)
    diag = lambda m: m.diagonal().cpu().numpy().astype(np.float64)
    ov = diag(boxes_pairwise(ta, tb, OVERLAP_BEV))
    iou_pw = diag(boxes_pairwise(ta, tb, IOU_BEV))
    iou_nms = diag(ops.boxes_iou_bev(ta.contiguous(), tb.contiguous()))
    iou3 = diag(boxes_pairwise(ta, tb, IOU_3D))
    iou3_al = boxes_iou3d_aligned(ta, tb).cpu().numpy().astype(np.float64)
    iou2 = diag(boxes_pairwise(ta, tb, IOU_2D))
    A, B = gr._f64(a), gr._f64(b)

    lo, hi = gr.exact_overlap(a, b), gr.exact_overlap(a, b, gr.MARGIN)
    ref, margin = gr.restated_overlap(a, b)
    bound = gr.overlap_bound(a, b)
    sure = margin > 1
    assert np.all(ov >= lo - bound), (family, np.max(lo - bound - ov))
    assert np.all(ov <= hi + bound), (family, np.max(ov - hi - bound))
    assert np.all(np.abs(ov - ref)[sure] <= bound[sure]), (family, np.max((np.abs(ov - ref) - bound)[sure]))
    far = gr.far_pair(a, b)
    assert np.all(ov[far] == 0), family

    # BEV IoU: the overlap's bound through so / max(Sa + Sb - so, 1e-8)
    S = A[:, 3] * A[:, 4] + B[:, 3] * B[:, 4]
    for name, got in (('iou_bev', iou_nms), ('pairwise IOU_BEV', iou_pw)):
        assert np.all(np.isfinite(got)) and np.all(got >= 0), (family, name)
        tol = _ratio_bound(ref, bound, S, 1e-8)
        assert np.all(np.abs(got - _ratio(ref, S, 1e-8))[sure] <= tol[sure]), (family, name)
        lo_i = _ratio(np.maximum(lo - bound, 0), S, 1e-8) - _ratio_bound(np.maximum(lo - bound, 0), 0, S, 1e-8)
        hi_i = _ratio(hi + bound, S, 1e-8) + _ratio_bound(hi + bound, 0, S, 1e-8)
        hi_i = np.where(S - hi - bound > 1e-8, hi_i, np.inf)     # a grown overlap that reaches the union bounds nothing
        assert np.all(got >= lo_i) and np.all(got <= hi_i), (family, name)

    # 3-D IoU: BEV overlap times the z overlap over the union volume, guarded by 1e-6; the z overlap rounds z +- h/2 (<= U *
    # (|z| + h/2) each), their min / max difference (<= U * oh): d_oh <= 3U * (|z| + h)
    za, zb = (A[:, 2] - A[:, 5] / 2, A[:, 2] + A[:, 5] / 2), (B[:, 2] - B[:, 5] / 2, B[:, 2] + B[:, 5] / 2)
    oh = np.maximum(np.minimum(za[1], zb[1]) - np.maximum(za[0], zb[0]), 0)
    d_oh = 3 * U * (np.maximum(np.abs(A[:, 2]), np.abs(B[:, 2])) + np.maximum(A[:, 5], B[:, 5]))
    V = A[:, 3] * A[:, 4] * A[:, 5] + B[:, 3] * B[:, 4] * B[:, 5]
    o3, d_o3 = ref * oh, bound * oh + (ref + bound) * d_oh + U * ref * oh
    for name, got in (('pairwise IOU_3D', iou3), ('iou3d_aligned', iou3_al)):
        assert np.all(np.isfinite(got)) and np.all(got >= 0), (family, name)
        tol = _ratio_bound(o3, d_o3, V, 1e-6)
        assert np.all(np.abs(got - _ratio(o3, V, 1e-6))[sure] <= tol[sure]), (family, name)
    # refine/score.boxes_iou3d_aligned promises the diagonal of the pairwise 3-D IoU, bit for bit
    assert np.array_equal(iou3_al.view(np.int64), iou3.view(np.int64)), family

    # axis-aligned 2-D IoU on (x, y, l, w): the edges x +- l/2 round by <= U * M, the overlap widths by <= U * iw: d_iw <= 3U * M
    M = np.maximum(np.abs(A[:, :2]).max(1) + A[:, 3:5].max(1), np.abs(B[:, :2]).max(1) + B[:, 3:5].max(1))
    iw = np.maximum(np.minimum(A[:, 0] + A[:, 3] / 2, B[:, 0] + B[:, 3] / 2) - np.maximum(A[:, 0] - A[:, 3] / 2, B[:, 0] - B[:, 3] / 2), 0)
    ih = np.maximum(np.minimum(A[:, 1] + A[:, 4] / 2, B[:, 1] + B[:, 4] / 2) - np.maximum(A[:, 1] - A[:, 4] / 2, B[:, 1] - B[:, 4] / 2), 0)
    inter, d_in = iw * ih, 3 * U * M * (iw + ih + 3 * U * M) + U * iw * ih
    ok2 = S > 0                                   # no union guard here (distance.py's IoU2D): two empty boxes give 0 / 0
    assert np.all(np.isnan(iou2[~ok2])), family
    tol = _ratio_bound(inter, d_in, S, 1e-30)[ok2]
    err = np.abs(iou2 - _ratio(inter, S, 1e-30))[ok2]
    assert np.all(err <= tol), (family, np.max(err - tol))


def test_iou_of_empty_boxes_is_guarded(cuda):
    """two zero-area boxes on top of each other: the 1e-8 / 1e-6 union guards keep the BEV and 3-D IoU finite"""
    a = np.array([[1, 2, 0, 0, 2, 1, 0.3], [1, 2, 0, 3, 0, 1, 0.0], [1, 2, 0, 0, 0, 1, 0.0]], np.float32)
    b = np.array([[1, 2, 0, 0, 2, 1, 1.2], [1.5, 2, 0, 3, 0, 1, 0.0], [1, 2, 0, 0, 0, 1, 0.0]], np.float32)
    ta, tb = _rows(a, cuda), _rows(b, cuda)
    for kind in (IOU_BEV, IOU_3D):
        got = boxes_pairwise(ta, tb, kind).cpu().numpy()
        assert np.all(np.isfinite(got)) and np.all(got >= 0), kind
    assert torch.all(torch.isfinite(ops.boxes_iou_bev(ta.contiguous(), tb.contiguous())))
    assert ops.boxes_iou_bev(ta[:0].contiguous(), tb.contiguous()).shape == (0, 3)          # an empty frame: an empty matrix


@pytest.mark.parametrize('family', ['random', 'identical', 'rot_k_half_pi', 'nested', 'pedestrian', 'heading_wrap', 'world_offset',
                                    'zero_size'])
def test_points_in_boxes_vs_float64(cuda, family):
    """dz_points_in_boxes_mask against the float64 test (|z - cz| <= h/2, |local x| < l/2 + 1e-5, |local y| < w/2 + 1e-5) on
    points placed on, just inside and just outside every face.  Only a point closer to a face than the test's rounding bound
    may differ: the local coordinates (x - cx) cos - (y - cy) sin round by <= 5U * (|dx| + |dy|) (subtraction, cosf / sinf at
    2 ulp, products, sum) and l/2 + 1e-5 by U * l; z - cz rounds by U * |z - cz|.  That is far inside the 1e-4 m the object crop
    test allows."""
    a, b = gr.pair_family(family, 96)
    boxes = np.concatenate([a, b])
    bx = gr._f64(boxes)
    g = np.random.default_rng(7)
    T, per = bx.shape[0], 24
    step = np.array([-1e-3, -3e-6, -1e-7, 0.0, 1e-7, 3e-6, 1e-3, 0.3])
    lx = (bx[:, 3:4] / 2 + np.float32(1e-5)) * g.choice([-1, 1], (T, per)) + g.choice(step, (T, per))
    ly = (bx[:, 4:5] / 2 + np.float32(1e-5)) * g.choice([-1, 1], (T, per)) + g.choice(step, (T, per))
    lz = bx[:, 5:6] / 2 * g.choice([-1, 1], (T, per)) + g.choice(step, (T, per))
    inner = g.random((T, per)) < 0.5                      # half the points: only one coordinate on a face
    lx = np.where(inner & (g.random((T, per)) < 0.5), lx * g.uniform(0, 1, (T, per)), lx)
    ly = np.where(inner & (g.random((T, per)) < 0.5), ly * g.uniform(0, 1, (T, per)), ly)
    c, s = np.cos(bx[:, 6:7]), np.sin(bx[:, 6:7])
    pts = np.stack([bx[:, 0:1] + lx * c - ly * s, bx[:, 1:2] + lx * s + ly * c, bx[:, 2:3] + lz], -1).reshape(-1, 3)
    pts = pts.astype(np.float32)
    got = points_in_boxes_gpu_v2(torch.from_numpy(pts)[None].to(cuda), torch.from_numpy(boxes)[None].to(cuda))[0].cpu().numpy()
    P = pts.astype(np.float64)
    dx, dy, dz = P[None, :, 0] - bx[:, 0:1], P[None, :, 1] - bx[:, 1:2], P[None, :, 2] - bx[:, 2:3]
    ca, sa = np.cos(-bx[:, 6:7]), np.sin(-bx[:, 6:7])
    rx, ry = dx * ca - dy * sa, dx * sa + dy * ca
    m5 = float(np.float32(1e-5))
    hx, hy, hz = bx[:, 3:4] / 2 + m5, bx[:, 4:5] / 2 + m5, bx[:, 5:6] / 2
    want = (np.abs(dz) <= hz) & (np.abs(rx) < hx) & (np.abs(ry) < hy)
    e_xy = 5 * U * (np.abs(dx) + np.abs(dy)) + U * np.maximum(bx[:, 3:4], bx[:, 4:5])
    near = (np.abs(np.abs(rx) - hx) <= e_xy) | (np.abs(np.abs(ry) - hy) <= e_xy) | (np.abs(np.abs(dz) - hz) <= U * np.abs(dz))
    diff = got.astype(bool) != want
    assert not np.any(diff & ~near), (family, int((diff & ~near).sum()))
    own = want.reshape(T, T, per)[np.arange(T), np.arange(T)]
    assert own.sum() > T * per // 20 and (~own).sum() > T * per // 20     # both sides of each box's faces are exercised


# ---- NMS ----------------------------------------------------------------------------------------------------------------
def _random_boxes(g, n, span=30.0):
    bx = np.concatenate([g.uniform(-span, span, (n, 2)), g.uniform(-1, 1, (n, 1)), g.uniform(0.5, 5, (n, 2)),
                         g.uniform(1, 2, (n, 1)), g.uniform(-np.pi, np.pi, (n, 1))], 1)
    k = n // 3                                            # clusters of near-duplicates, as the head's neighbouring cells give
    bx[n - k:, :2] = bx[:k, :2] + g.normal(0, 0.4, (k, 2))
    bx[n - k:, 3:7] = bx[:k, 3:7] + g.normal(0, 0.05, (k, 4))
    bx[:, 3:5] = np.abs(bx[:, 3:5]) + 0.1
    return bx.astype(np.float32)


def _iou_matrix(boxes, cuda):
    t = torch.from_numpy(boxes).to(cuda)
    return ops.boxes_iou_bev(t, t).cpu().numpy()


def _away_from(boxes, thresh, cuda):
    """grow boxes until every IoU of a pair (i < j) lies >= 1e-5 from the threshold: the mask kernel and the IoU kernel may round
    the same IoU differently (separate kernels, separate FMA contraction), by far less than that.  (Exact cases -- identical and
    disjoint boxes -- are built by the tests that need them.)"""
    boxes = boxes.copy()
    for _ in range(20):
        iou = _iou_matrix(boxes, cuda)
        close = np.triu(np.abs(iou - thresh) < 1e-5, 1)
        if not close.any():
            return boxes
        boxes[np.nonzero(close)[1], 3] *= np.float32(1.01)
    raise AssertionError('could not move the test boxes away from the NMS threshold')


def _greedy_nms(iou, thresh):
    """the reference keep scan over a given IoU matrix: box i survives unless a kept box before it has IoU > thresh with it"""
    n = iou.shape[0]
    removed = np.zeros(n, bool)
    keep = []
    for i in range(n):
        if removed[i]:
            continue
        keep.append(i)
        removed[i + 1:] |= iou[i, i + 1:] > thresh
    return np.array(keep, np.int64)


def _run_nms(cuda, frames, cap, d_n, thresh, post_max, label_offset, seed):
    """frames: list of (n_b, 7) boxes; d_n may exceed cap (clamped by the kernels).  Output written into views of larger
    buffers whose surroundings must stay untouched."""
    B = len(frames)
    g = np.random.default_rng(seed)
    pb = np.zeros((B, cap, 7), np.float32)
    ps = np.zeros((B, cap), np.float32)
    pl = g.integers(0, 3, (B, cap)).astype(np.int32)
    for k, f in enumerate(frames):
        pb[k, :len(f)] = f[:cap]
        ps[k, :min(len(f), cap)] = np.sort(g.uniform(0.05, 1, min(len(f), cap)).astype(np.float32))[::-1]
    big = torch.full((B + 2, post_max, 9), -5.0, dtype=torch.float32, device=cuda)
    big_n = torch.full((B + 3,), -9, dtype=torch.int32, device=cuda)
    out, d_out = big[1:1 + B], big_n[2:2 + B]
    ops.nms_bev(torch.from_numpy(pb).to(cuda), torch.from_numpy(ps).to(cuda), torch.from_numpy(pl).to(cuda),
                torch.tensor(d_n, dtype=torch.int32, device=cuda), thresh, post_max, label_offset=label_offset, out=out,
                d_out_n=d_out)
    assert torch.all(big[0] == -5.0) and torch.all(big[B + 1] == -5.0)
    assert torch.all(big_n[:2] == -9) and torch.all(big_n[2 + B:] == -9)
    return pb, ps, pl, out.cpu().numpy(), d_out.cpu().numpy()


def _check_nms(cuda, frames, cap, d_n, thresh, post_max, label_offset=1, seed=0):
    pb, ps, pl, out, d_out = _run_nms(cuda, frames, cap, d_n, thresh, post_max, label_offset, seed)
    kept = []
    for k in range(len(frames)):
        n = min(d_n[k], cap)
        keep = _greedy_nms(_iou_matrix(pb[k, :n], cuda), thresh) if n else np.zeros(0, np.int64)
        m = min(len(keep), post_max)
        assert d_out[k] == m, (k, d_out[k], m)
        keep = keep[:m]
        assert np.array_equal(out[k, :m, :7], pb[k, keep]), k
        assert np.array_equal(out[k, :m, 7], ps[k, keep]), k
        assert np.array_equal(out[k, :m, 8], (pl[k, keep] + label_offset).astype(np.float32)), k
        assert np.all(out[k, m:] == 0), k                 # rows past the kept count: exactly zero
        kept.append(keep)
    return kept


# (cap, n per frame): every n of {0, 1, 63, 64, 65, 127, 128, 129, 500} at B = 3 next to 64-box block boundaries, the capacities
# {1, 64, 65, 500, 1024, 1248}, and counts above the capacity (clamped to it)
NMS_CASES = [(1, (0, 1, 5)), (64, (63, 64, 100)), (65, (65, 1, 64)), (500, (127, 128, 129)), (500, (500, 0, 65)),
             (1024, (500, 129, 1024)), (1248, (1248, 64, 0))]


@pytest.mark.parametrize('cap,ns', NMS_CASES, ids=['cap%d-%s' % (c, '-'.join(map(str, n))) for c, n in NMS_CASES])
def test_nms_vs_greedy_over_kernel_iou(cuda, cap, ns):
    """device NMS == greedy NMS over the kernel's own IoU matrix, per frame, for post_max below the kept count and above n, two
    label offsets, outputs written into views"""
    g = np.random.default_rng(cap + sum(ns))
    thresh = 0.3
    frames = [_away_from(_random_boxes(g, min(n, cap)), thresh, cuda) for n in ns]
    for post_max, off in ((3, 1), (max(ns) + 7, 0), (max(ns) + 7, 4)):
        kept = _check_nms(cuda, frames, cap, list(ns), thresh, post_max, label_offset=off, seed=cap)
    assert cap < 4 or any(len(k) > 3 for k in kept)        # post_max = 3 cut some frame short


@pytest.mark.parametrize('start,n,cap', [(0, 40, 64), (0, 200, 256), (1, 200, 256), (1, 130, 1248)])
def test_nms_suppression_chain(cuda, start, n, cap):
    """boxes on a line where box i overlaps only box i+1 (IoU 0.5 / 3.5 = 0.14 > 0.1; two apart they are 1 m apart, IoU exactly
    0): every other box is kept, because a suppressed box suppresses nothing.  `start` isolated boxes come first; with one, box
    63 is kept and must remove box 64 across the 64-box block boundary."""
    bx = np.zeros((n, 7), np.float32)
    bx[:, 0] = (np.arange(n) - start) * 1.5
    bx[:start, 0] = -400.0 - 10.0 * np.arange(start)
    bx[:, 1], bx[:, 3], bx[:, 4], bx[:, 5] = 3.0, 2.0, 1.0, 1.5
    kept = _check_nms(cuda, [bx], cap, [n], 0.1, n + 1)[0]
    assert np.array_equal(kept, np.concatenate([np.arange(start), np.arange(start, n, 2)]))


def test_nms_identical_and_disjoint_boxes(cuda):
    """exact cases: n identical boxes keep exactly one; disjoint boxes (IoU exactly 0) all survive a threshold of 0 (strict >),
    at B = 2 with the two frames in one call"""
    same = np.tile(np.array([[3, 4, 0.5, 4.2, 1.9, 1.6, 0.7]], np.float32), (300, 1))
    grid = np.stack(np.meshgrid(np.arange(20) * 8.0, np.arange(15) * 8.0), -1).reshape(-1, 2)
    disj = np.concatenate([grid, np.zeros((300, 1)), np.full((300, 2), 3.0), np.ones((300, 1)),
                           np.random.default_rng(1).uniform(-np.pi, np.pi, (300, 1))], 1).astype(np.float32)
    kept = _check_nms(cuda, [same, disj], 320, [300, 300], 0.0, 310)
    assert len(kept[0]) == 1 and len(kept[1]) == 300


def test_nms_rejects_a_cap_over_the_scan_limit_without_launching(cuda):
    """1248 is the largest cap whose mask + keep list fit the scan's 200 KB of shared memory; 1249 returns DZ_ERR_UNSUPPORTED
    before anything is enqueued: the workspace and the outputs are left as they were"""
    L = _lib.lib()
    assert 1248 * 20 * 8 + 1248 * 4 <= 200 * 1024 < 1249 * 20 * 8 + 1249 * 4
    cap, B, post_max = 1249, 1, 16
    g = np.random.default_rng(3)
    boxes = torch.zeros((B, cap, 7), dtype=torch.float32, device=cuda)
    boxes[0, :200] = torch.from_numpy(_random_boxes(g, 200)).to(cuda)
    scores = torch.zeros((B, cap), dtype=torch.float32, device=cuda)
    labels = torch.zeros((B, cap), dtype=torch.int32, device=cuda)
    d_n = torch.tensor([200], dtype=torch.int32, device=cuda)
    nbytes = L.dz_nms_bev_ws_bytes(B, cap)
    ws = torch.full((nbytes,), 0x5A, dtype=torch.uint8, device=cuda)
    out = torch.full((B, post_max, 9), -5.0, dtype=torch.float32, device=cuda)
    d_out = torch.full((B,), -9, dtype=torch.int32, device=cuda)
    rc = L.dz_nms_bev(ops._p(boxes), ops._p(scores), ops._p(labels), ops._p(d_n), B, cap, ctypes.c_float(0.5), post_max, 1,
                      ops._p(out), ops._p(d_out), ops._p(ws), nbytes, ops._stream())
    torch.cuda.synchronize()
    assert rc == -4                                       # DZ_ERR_UNSUPPORTED
    assert torch.all(ws == 0x5A) and torch.all(out == -5.0) and torch.all(d_out == -9)


# ---- CenterHead decode --------------------------------------------------------------------------------------------------
# channel layout of the test head maps: center 2, center_z 1, dim 3, rot 2 (cos, sin), iou 1, hm num_class
LAYOUT = {'center': 0, 'center_z': 2, 'dim': 3, 'rot': 6, 'iou': 8, 'hm': 9}
PC_RANGE = [-75.2, -75.2, -2.0, 75.2, 75.2, 4.0]
VOXEL = [0.1, 0.1, 0.15]
STRIDE = 8
WIDE = [-1e4, -1e4, -1.0, 1e4, 1e4, 1e7]                  # post-centre limits that keep every box (z carries the pixel index)
SIG_BOUND = 8 * U
"""score bound, relative: expf(-x) at 2 ulp (<= 4U), 1 + e and 1 / (1 + e) one rounding each, clamp(iou)^2 and the product one
rounding each: |s - sigmoid(x) * q^2| <= 8U * s"""


def _head_maps(g, B, H, W, C, tie_frac=0.4, sat_frac=0.02, zero_iou_frac=0.1):
    """random head maps with exact ties (logits and ious drawn from small pools, across pixels and classes), saturated
    sigmoids (logit 30: sigmoid == 1.0 in float32), ious <= 0 (score +0) and continuous values; center_z = pixel index"""
    HW = H * W
    h = np.zeros((B, HW, 9 + C), np.float32)
    h[..., 0:2] = g.uniform(0, 1, (B, HW, 2))
    h[..., 2] = np.arange(HW)
    h[..., 3:6] = g.normal(0.3, 0.6, (B, HW, 3))
    h[..., 6:8] = g.normal(0, 1, (B, HW, 2))
    iou = g.uniform(-0.2, 1.2, (B, HW))
    pool = g.random((B, HW))
    iou = np.where(pool < tie_frac, g.choice([0.5, 0.75, 1.0], (B, HW)), iou)
    iou = np.where(pool > 1 - zero_iou_frac, g.choice([0.0, -0.3], (B, HW)), iou)
    h[..., 8] = iou
    hm = g.normal(-2, 2, (B, HW, C))
    pick = g.random((B, HW, C))
    hm = np.where(pick < tie_frac, g.choice([-1.0, 0.5, 1.25, 2.0], (B, HW, C)), hm)
    hm = np.where(pick > 1 - sat_frac, 30.0, hm)
    h[..., 9:] = hm
    return h.reshape(B, H, W, 9 + C)


def _decode_ref(head, C, K, thresh, use_iou, limit):
    """float64 decode per frame: (selected [t], ambiguous set {t}, score, score bound, box, box bound), elements t = cls * HW +
    pixel.  Order: score descending, then class-major (the merged list is flattened class by class), then pixel index ascending;
    top K; then the post-centre limits (inclusive) and score > threshold (strict), order kept.  Ambiguous: an element that may
    land on the other side of the K boundary, the threshold or a limit because its float64 value is within the rounding bounds
    of it -- never an exact tie, which the kernel must break like the reference."""
    B, H, W, ch = head.shape
    HW = H * W
    hd = head.reshape(B, HW, ch).astype(np.float64)
    lo = np.float32(PC_RANGE[:3]).astype(np.float64)
    vs = np.float32(VOXEL).astype(np.float64)
    lim = np.float32(limit).astype(np.float64)
    th = np.float64(np.float32(thresh))
    cls, idx = np.repeat(np.arange(C), HW), np.tile(np.arange(HW), C)
    res = []
    for b in range(B):
        s = 1.0 / (1.0 + np.exp(-hd[b, :, 9:9 + C]))
        if use_iou:
            s = s * np.clip(hd[b, :, 8], 0, 1)[:, None] ** 2
        sv = s.T.reshape(-1)
        sb = SIG_BOUND * sv
        order = np.lexsort((idx, cls, -sv))
        top, rest = order[:min(K, C * HW)], order[min(K, C * HW):]
        amb = set()
        if len(rest):                                     # the K boundary
            near_in = top[sv[top] <= sv[top[-1]] * (1 + 2 * SIG_BOUND)]
            near_out = rest[sv[rest] >= sv[rest[0]] * (1 - 2 * SIG_BOUND)]
            for x in np.unique(sv[near_in]):
                for y in np.unique(sv[near_out]):
                    if x != y and abs(x - y) <= SIG_BOUND * (x + y):
                        amb |= set(near_in[sv[near_in] == x].tolist()) | set(near_out[sv[near_out] == y].tolist())
        ix, iy = idx % W, idx // W
        xs = (ix + hd[b, idx, 0]).astype(np.float32).astype(np.float64)          # (float)(idx % W) + center: one rounding
        ys = (iy + hd[b, idx, 1]).astype(np.float32).astype(np.float64)
        box = np.stack([xs * STRIDE * vs[0] + lo[0], ys * STRIDE * vs[1] + lo[1], hd[b, idx, 2], np.exp(hd[b, idx, 3]),
                        np.exp(hd[b, idx, 4]), np.exp(hd[b, idx, 5]), np.arctan2(hd[b, idx, 7], hd[b, idx, 6])], 1)
        # x, y: fl(ix + cx), * stride, * voxel, + lo: 3 roundings of |xs * stride * vs| and one of |x|; z copied; expf 2 ulp;
        # atan2f 3 ulp
        bb = np.stack([3 * U * np.abs(xs * STRIDE * vs[0]) + U * np.abs(box[:, 0]),
                       3 * U * np.abs(ys * STRIDE * vs[1]) + U * np.abs(box[:, 1]), np.zeros(len(idx)),
                       4 * U * box[:, 3], 4 * U * box[:, 4], 4 * U * box[:, 5], 6 * U * np.abs(box[:, 6])], 1)
        inside = np.ones(len(idx), bool)
        near = np.abs(sv - th) <= sb
        for d in range(3):
            inside &= (box[:, d] >= lim[d]) & (box[:, d] <= lim[d + 3])
            near |= (np.abs(box[:, d] - lim[d]) <= bb[:, d]) | (np.abs(box[:, d] - lim[d + 3]) <= bb[:, d])
        exact = (sv == th) | np.any(box[:, :3] == lim[None, :3], 1) | np.any(box[:, :3] == lim[None, 3:], 1)
        amb |= set(top[(near & ~exact)[top]].tolist())
        sel = top[inside[top] & (sv[top] > th)]
        res.append((sel, amb, sv, sb, box, bb))
    return res


def _check_decode(cuda, head, C, K, thresh, use_iou, limit=WIDE):
    boxes, scores, labels, d_n = ops.centerhead_decode(torch.from_numpy(head).to(cuda), LAYOUT, C, K, PC_RANGE, VOXEL, STRIDE,
                                                       limit, thresh, use_iou)
    boxes, scores, labels, d_n = boxes.cpu().numpy(), scores.cpu().numpy(), labels.cpu().numpy(), d_n.cpu().numpy()
    HW = head.shape[1] * head.shape[2]
    ref = _decode_ref(head, C, K, thresh, use_iou, limit)
    for b, (want, amb, sv, sb, box, bb) in enumerate(ref):
        n = int(d_n[b])
        got = labels[b, :n].astype(np.int64) * HW + boxes[b, :n, 2].astype(np.int64)     # center_z carries the pixel index
        assert len(set(got.tolist())) == n, b
        assert set(got.tolist()) ^ set(want.tolist()) <= amb, (b, sorted(set(got.tolist()) ^ set(want.tolist()) - amb)[:5])
        # the kernel's own order: its score descending, ties by class, then by pixel index (= by t)
        key = list(zip((-scores[b, :n]).tolist(), got.tolist()))
        assert key == sorted(key), b
        err = np.abs(scores[b, :n].astype(np.float64) - sv[got])
        assert np.all(err <= sb[got]), (b, np.max(err - sb[got]))
        berr = np.abs(boxes[b, :n].astype(np.float64) - box[got])
        assert np.all(berr <= bb[got]), (b, np.max(berr - bb[got], 0))
    return ref, scores, d_n


DECODE_CASES = {                  # B, H, W, num_class, K, threshold, use_iou
    'K1': (4, 40, 36, 3, 1, 0.05, True),
    'K7': (4, 40, 36, 3, 7, 0.05, True),
    'K500': (4, 48, 40, 3, 500, 0.1, True),
    'K1024-C4': (2, 64, 72, 4, 1024, 0.05, True),          # num_class * K = 4096, the merge's limit
    'HW-below-K': (3, 8, 8, 3, 500, 0.05, True),
    'HW-below-K-negative-threshold': (3, 8, 8, 3, 500, -1.0, True),
    'negative-threshold': (2, 16, 16, 3, 700, -0.5, True),  # full-map select; K cuts through the +0 scores, which tie across
                                                            # classes and pixels
    'no-iou': (4, 48, 40, 3, 500, 0.1, False),
}


@pytest.mark.parametrize('case', list(DECODE_CASES))
def test_decode_vs_float64(cuda, case):
    B, H, W, C, K, thresh, use_iou = DECODE_CASES[case]
    g = np.random.default_rng(len(case) * 7 + K)
    head = _head_maps(g, B, H, W, C)
    ref, scores, d_n = _check_decode(cuda, head, C, K, thresh, use_iou)
    assert any(len(r[0]) for r in ref)
    if use_iou and thresh < 0:                            # +0 scores were selected: the ties at 0 went by class and index
        assert any(np.any(scores[b, :d_n[b]] == 0) for b in range(B))
    if case == 'K500':
        assert np.any(scores == 1.0)                      # saturated sigmoids tie at exactly 1.0


@pytest.mark.parametrize('n_above', [4095, 4096, 4097])
def test_decode_candidate_list_switch(cuda, n_above):
    """exactly 4095 / 4096 / 4097 scores above the threshold in one (frame, class): the candidate list holds up to 4096 (fast
    path), one more sends that (frame, class) to the full-map radix select; K falls among exact ties"""
    B, H, W, C, K, thresh = 2, 80, 80, 3, 500, 0.1
    g = np.random.default_rng(n_above)
    head = _head_maps(g, B, H, W, C, zero_iou_frac=0.0)
    hw = H * W
    flat = head.reshape(B, hw, -1)
    pick = g.permutation(hw)[:n_above]
    flat[0, :, 9] = g.uniform(-12, -6, hw)                # sigmoid <= 2.5e-3: below the threshold
    flat[0, pick, 9] = g.choice([1.5, 2.0, 2.5], n_above)  # sigmoid >= 0.81 ...
    flat[0, :, 8] = g.choice([0.75, 1.0], hw)             # ... times >= 0.56: above it, in 6 exact tie groups
    flat[0, pick[:5], 9] = 30.0
    ref, scores, d_n = _check_decode(cuda, head, C, K, thresh, True)
    s = 1 / (1 + np.exp(-flat[0, :, 9].astype(np.float64))) * np.clip(flat[0, :, 8], 0, 1) ** 2
    assert int((s > thresh).sum()) == n_above and np.all(np.abs(s - thresh) > 0.05)
    assert d_n[0] == K


def test_decode_threshold_and_limits_are_exact(cuda):
    """a score exactly equal to the threshold is dropped (strict >); centres exactly on the post-centre limits are kept
    (inclusive), just past them dropped.  All of it is exact in float32: sigmoid(30) == 1.0 (expf(-30) < 2^-25 vanishes in
    1 + e), times 0.5^2; centres (ix + cx) * 8 * 0.125 - 16 with dyadic offsets, z copied."""
    B, H, W, C, K = 1, 32, 32, 2, 500
    g = np.random.default_rng(5)
    head = _head_maps(g, B, H, W, C, zero_iou_frac=0.0)
    flat = head.reshape(B, H * W, -1)
    flat[..., 0:2] = g.choice([0.0, 0.25, 0.5, 0.75], flat[..., 0:2].shape)
    flat[..., 2] = g.choice([-2.0, -1.5, 0.0, 3.0, 3.25, -2.25], H * W)
    flat[..., 9:] = g.choice([-20.0, 30.0], flat[..., 9:].shape, p=[0.5, 0.5])
    flat[..., 8] = g.choice([0.5, 1.0, 0.25], H * W)      # scores 0.25 (== threshold), 1.0, 0.0625
    limit = [-10.0, -9.75, -2.0, 10.0, 9.5, 3.0]
    pc = [-16.0, -16.0, -2.0, 16.0, 16.0, 4.0]
    vs = [0.125, 0.125, 0.15]
    boxes, scores, labels, d_n = ops.centerhead_decode(torch.from_numpy(head).to(cuda), LAYOUT, C, K, pc, vs, STRIDE, limit,
                                                       0.25, True)
    n = int(d_n[0])
    hw = np.arange(H * W)
    x = (hw % W + flat[0, :, 0].astype(np.float64)) * STRIDE * 0.125 - 16
    y = (hw // W + flat[0, :, 1].astype(np.float64)) * STRIDE * 0.125 - 16
    z = flat[0, :, 2].astype(np.float64)
    keep_pix = (x >= -10) & (x <= 10) & (y >= -9.75) & (y <= 9.5) & (z >= -2) & (z <= 3) & (flat[0, :, 8] == 1.0)
    want = sorted((c, i) for c in range(C) for i in np.nonzero(keep_pix & (flat[0, :, 9 + c] == 30.0))[0])
    assert len(want) < K
    got_xyz = boxes[0, :n, :3].cpu().numpy().astype(np.float64)
    got_lab = labels[0, :n].cpu().numpy()
    assert np.all(scores[0, :n].cpu().numpy() == 1.0)
    # identify each output by its exact centre (x, y identify the pixel, z is exact) and its label
    pix = {(x[i], y[i], z[i]): i for i in np.nonzero(keep_pix)[0]}
    got = sorted((int(got_lab[r]), pix[tuple(got_xyz[r])]) for r in range(n))
    assert got == want
    on_edge = [(x[i] in (-10, 10)) or (y[i] in (-9.75, 9.5)) or (z[i] in (-2, 3)) for _, i in want]
    assert any(on_edge)
    out_by_a_step = (np.isin(x, [-10.25, 10.25]) | np.isin(y, [-10.0, 9.75]) | np.isin(z, [-2.25, 3.25])) & (flat[0, :, 8] == 1.0)
    assert out_by_a_step.any()

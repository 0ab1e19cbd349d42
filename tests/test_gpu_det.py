"""GPU parity tests for the detector hot path: every kernel of libdetzero_b200 against the CPU oracle on the same
seeded inputs (SURVEY.md §8c parity definitions).  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest
import torch

import oracle
from oracle import det_ref, spconv_ref, weights
from tests import spconv_arith as sa
from tests import util
from detzero_b200 import _lib

pytestmark = pytest.mark.gpu


def _pairs_from_nbr(nbr, n_out):
    """neighbour table (K, cap) -> set of (k, in, out)"""
    nbr = nbr[:, :n_out].cpu().numpy()
    k, o = np.nonzero(nbr >= 0)
    return set(zip(k.tolist(), nbr[k, o].tolist(), o.tolist()))


def _pairs_from_oracle(pairs):
    s = set()
    for k, (i_in, i_out) in enumerate(pairs):
        s.update(zip([k] * len(i_in), np.asarray(i_in).tolist(), np.asarray(i_out).tolist()))
    return s


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n,max_voxels,rng_', [(20000, 200000, util.WAYMO_RANGE), (20000, 3000, util.WAYMO_RANGE),
                                               (50000, 200000, util.SMALL_RANGE), (0, 100, util.WAYMO_RANGE),
                                               (7, 100, util.WAYMO_RANGE)])
def test_voxelize_hard_bit_exact(cuda, n, max_voxels, rng_):
    """BASELINE config[0]: voxel coords / counts / order / features bit-exact vs the CPU voxelizer"""
    from detzero_b200.spconv.utils import Point2VoxelGPU3d
    pts = util.config1_cloud(n, seed=1, pc_range=rng_) if n else np.zeros((0, 5), np.float32)
    if rng_ is util.SMALL_RANGE:
        pts = np.concatenate([pts, util.clustered_cloud(n, 3)], axis=0)
    ref = oracle.Point2VoxelCPU3d(util.VOXEL, rng_, 5, 5, max_voxels)
    rv, rc, rn = ref.point_to_voxel(pts)
    gen = Point2VoxelGPU3d(util.VOXEL, rng_, 5, 5, max_voxels, device=cuda)
    v, c, m = gen.point_to_voxel(torch.from_numpy(pts).to(cuda))
    assert v.shape[0] == rv.shape[0]
    assert np.array_equal(c.cpu().numpy(), rc)
    assert np.array_equal(m.cpu().numpy(), rn)
    assert np.array_equal(v.cpu().numpy().view(np.uint32), rv.view(np.uint32))      # bit-exact features


def test_voxelize_batch_and_mean(cuda):
    from detzero_b200.spconv.utils import Point2VoxelGPU3d
    clouds = [util.clustered_cloud(30000, 5), util.config1_cloud(10000, 6, util.SMALL_RANGE), util.clustered_cloud(500, 7)]
    gen = Point2VoxelGPU3d(util.VOXEL, util.SMALL_RANGE, 5, 5, 20000, device=cuda)
    pts_b = [torch.from_numpy(np.pad(p, ((0, 0), (1, 0)), constant_values=b)).to(cuda) for b, p in enumerate(clouds)]
    r = gen.voxelize_batch(pts_b, xyz_off=1)
    m = int(r['counters'][0].item())
    ref = oracle.Point2VoxelCPU3d(util.VOXEL, util.SMALL_RANGE, 5, 5, 20000)
    rv, rc, rn = [], [], []
    for b, p in enumerate(clouds):
        v, c, n = ref.point_to_voxel(p)
        rv.append(v); rn.append(n); rc.append(np.pad(c, ((0, 0), (1, 0)), constant_values=b))
    rv, rc, rn = np.concatenate(rv), np.concatenate(rc), np.concatenate(rn)
    assert m == rv.shape[0]
    assert np.array_equal(r['coords'][:m].cpu().numpy(), rc)
    assert np.array_equal(r['num'][:m].cpu().numpy(), rn)
    assert np.array_equal(r['voxels'][:m].cpu().numpy().view(np.uint32), rv.view(np.uint32))
    mean_ref = det_ref.mean_vfe(rv, rn)
    assert util.rel_err(r['mean'][:m].cpu(), mean_ref) < 1e-6
    # the index handed to the backbone resolves every voxel to its own row
    from detzero_b200 import ops
    nbr = ops.rulebook_subm(r['coords'], r['counters'][0:1], r['cap'], r['index'], [1, 1, 1])
    assert torch.equal(nbr[0, :m].cpu(), torch.arange(m, dtype=torch.int32))
    # MeanVFE on pre-voxelized input (reference contract)
    out = ops.mean_vfe(torch.from_numpy(rv).to(cuda), torch.from_numpy(rn).to(cuda))
    assert util.rel_err(out.cpu(), mean_ref) < 1e-6


def test_dynamic_mean_vfe(cuda):
    from detzero_b200 import ops
    clouds = [util.clustered_cloud(40000, 11, c=6), util.config1_cloud(15000, 12, util.SMALL_RANGE, c=6)]
    pts = np.concatenate([np.pad(p, ((0, 0), (1, 0)), constant_values=b) for b, p in enumerate(clouds)]).astype(np.float32)
    grid = [192, 192, 40]
    mean_ref, coords_ref = det_ref.dynamic_mean_vfe(pts, util.SMALL_RANGE, util.VOXEL, grid)
    feats, coords, d_m = ops.voxelize_dynamic_mean(torch.from_numpy(pts).to(cuda), 6, 2, util.SMALL_RANGE, util.VOXEL, grid, 60000)
    m = int(d_m.item())
    assert m == coords_ref.shape[0]
    assert torch.equal(coords[:m].cpu(), coords_ref)                       # order = ascending (b,x,y,z) key
    assert np.array_equal(feats[:m].cpu().numpy().view(np.uint32), mean_ref.numpy().view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------
def _sparse_input(cuda, seed, B, shape, density, cin):
    idx = weights.random_sparse_coords(seed, B, shape, density)
    f = torch.from_numpy(np.random.default_rng(seed + 1).normal(0, 1, (len(idx), cin)).astype(np.float32))
    return idx, f


@pytest.mark.parametrize('ks,stride,pad', [(3, 1, 1), (3, 2, 1), (3, 2, (0, 1, 1)), ((3, 1, 1), (2, 1, 1), 0)])
def test_rulebook_set_exact(cuda, ks, stride, pad):
    from detzero_b200 import ops
    from detzero_b200.spconv.pytorch import SparseConvTensor, _triple
    shape, B = [11, 40, 36], 2
    idx, f = _sparse_input(cuda, 21, B, shape, 0.08, 16)
    t = SparseConvTensor(f.to(cuda), torch.from_numpy(idx).to(cuda), shape, B)
    n = len(idx)
    if stride == 1:
        nbr = ops.rulebook_subm(t._idx, t._count, t._cap, t.grid_index(), _triple(ks))
        got = _pairs_from_nbr(nbr, n)
        want = _pairs_from_oracle(spconv_ref.rulebook_subm(idx, shape, ks))
        assert got == want
    else:
        oc, d_n, oi, nbr, odhw = ops.rulebook_conv(t._idx, t._count, t._cap, t.grid_index(), _triple(ks), _triple(stride),
                                                   _triple(pad), out_cap=n * 2)
        ref_idx, ref_shape, ref_pairs = spconv_ref.rulebook_conv(idx, shape, ks, stride, pad)
        m = int(d_n.item())
        assert odhw == ref_shape and m == ref_idx.shape[0]
        assert np.array_equal(oc[:m].cpu().numpy(), ref_idx)                # sorted (b,z,y,x): bit-exact site list
        assert _pairs_from_nbr(nbr, m) == _pairs_from_oracle(ref_pairs)


def test_rulebooks_on_an_overflowed_level_stay_inside_its_capacity(cuda):
    """a strided conv whose output capacity is below its site count keeps the first `cap` sites (ascending order) and reports the
    full count; the rulebooks built on that level (submanifold, and the next strided conv) must only name rows < cap: the sites
    past the capacity are in the level's grid index but have no row.  Otherwise the conv gathers outside the feature buffer."""
    from detzero_b200 import ops
    from detzero_b200.spconv.pytorch import SparseConvTensor
    shape, B = [11, 40, 36], 2
    idx, f = _sparse_input(cuda, 23, B, shape, 0.08, 16)
    t = SparseConvTensor(f.to(cuda), torch.from_numpy(idx).to(cuda), shape, B)
    ref_idx, ref_shape, _ = spconv_ref.rulebook_conv(idx, shape, 3, 2, 1)
    m = ref_idx.shape[0]
    cap = m // 2
    for layout in ('k', 'row'):
        oc, d_n, oi, tab, odhw = ops.rulebook_conv(t._idx, t._count, t._cap, t.grid_index(), [3, 3, 3], [2, 2, 2], [1, 1, 1],
                                                   out_cap=cap, layout=layout)
        assert int(d_n.item()) == m                                          # the overflow stays visible
        assert np.array_equal(oc.cpu().numpy(), ref_idx[:cap])
        # submanifold rulebook on the truncated level: the oracle's pairs among its first `cap` sites, nothing else
        nbr = ops.rulebook_subm(oc, d_n, cap, oi, [3, 3, 3], layout=layout)
        k_major = nbr if layout == 'k' else nbr[:, :27].t()
        want = {(k, i, o) for k, i, o in _pairs_from_oracle(spconv_ref.rulebook_subm(ref_idx, ref_shape, 3)) if i < cap and o < cap}
        assert int(k_major.max().item()) < cap
        assert _pairs_from_nbr(k_major.contiguous(), cap) == want, layout
        # the next strided conv reads the truncated level through the same index
        oc2, d_n2, _, nbr2, _ = ops.rulebook_conv(oc, d_n, cap, oi, [3, 3, 3], [2, 2, 2], [1, 1, 1], out_cap=4 * m, layout=layout)
        m2 = int(d_n2.item())
        k2 = nbr2[:, :m2] if layout == 'k' else nbr2[:m2, :27].t()
        ref2_idx, _, ref2_pairs = spconv_ref.rulebook_conv(ref_idx[:cap], ref_shape, 3, 2, 1)
        assert np.array_equal(oc2[:m2].cpu().numpy(), ref2_idx)
        assert int(k2.max().item()) < cap
        assert _pairs_from_nbr(k2.contiguous(), m2) == _pairs_from_oracle(ref2_pairs), layout


@pytest.mark.parametrize('cin,cout', [(5, 16), (16, 16), (16, 32), (32, 32), (32, 64), (64, 64), (64, 128), (128, 128)])
def test_spconv_fwd_fp32(cuda, cin, cout):
    """fp32-exact mode: <= 1e-5 rel (summation order only), with the fused affine/residual/ReLU epilogue"""
    from detzero_b200 import ops
    from detzero_b200.spconv.pytorch import SparseConvTensor
    shape, B = [9, 30, 30], 2
    idx, f = _sparse_input(cuda, 31 + cin, B, shape, 0.12, cin)
    n = len(idx)
    g = np.random.default_rng(5)
    w = torch.from_numpy(g.normal(0, 0.2, (cout, 3, 3, 3, cin)).astype(np.float32))
    scale = torch.from_numpy(g.uniform(0.5, 1.5, cout).astype(np.float32))
    shift = torch.from_numpy(g.normal(0, 0.1, cout).astype(np.float32))
    res = torch.from_numpy(g.normal(0, 1, (n, cout)).astype(np.float32))
    ref = spconv_ref.sparse_conv_native(f, w, spconv_ref.rulebook_subm(idx, shape, 3), n)
    ref = torch.relu(ref * scale + shift + res)
    t = SparseConvTensor(f.to(cuda), torch.from_numpy(idx).to(cuda), shape, B)
    nbr = ops.rulebook_subm(t._idx, t._count, t._cap, t.grid_index(), [3, 3, 3])
    for mode, tol in ((_lib.DZ_F32, 1e-5), (_lib.DZ_TF32, 2e-3), (_lib.DZ_TF32X3, 2e-5)):     # x3: bounded by the tensor core's fp32 accumulate
        wp = ops.pack_spconv_weight(w, mode).to(cuda)
        out = ops.spconv_fwd(t._feat, nbr, t._count, n, wp, scale.to(cuda), shift.to(cuda), res.to(cuda), True, mode,
                             kshape=(27, cin, cout))
        assert util.rel_err(out.cpu(), ref) < tol, mode
    # bf16 operand planes (persistent wgmma kernel): 2 planes = fp32-level, 1 plane = bf16 storage
    tab = ops.table_to_rows(nbr)
    cin_pad = 8 if cin <= 8 else cin
    for mode, tol in ((_lib.DZ_BF16X2, 2e-5), (_lib.DZ_BF16, 1e-2)):
        P = _lib.PLANES[mode]
        wp = ops.pack_spconv_weight(w, mode).to(cuda)
        fp = ops.to_planes(t._feat, t._count, P, cin_pad)
        rp = ops.to_planes(res.to(cuda), t._count, P)
        out = ops.spconv_fwd(fp, tab, t._count, n, wp, scale.to(cuda), shift.to(cuda), rp, True, mode, kshape=(27, cin, cout), layout='row')
        assert out.dtype == torch.bfloat16 and out.shape == (n, P * cout)
        assert util.rel_err(ops.from_planes(out, t._count, P).cpu(), ref) < tol, mode


def test_planes_roundtrip(cuda):
    """fp32 <-> bf16 operand planes: p0 = RN_bf16(x), p1 = RN_bf16(x - p0); 2 planes keep 16 significand bits, channels are
    zero-padded, rows beyond the device count are left alone"""
    from detzero_b200 import ops
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(1000, 5, generator=g) * torch.logspace(-3, 3, 1000)[:, None]).to(cuda)
    d_n = torch.tensor([900], dtype=torch.int32, device=cuda)
    for P in (1, 2):
        pl = ops.to_planes(x, d_n, P, 8)
        assert pl.shape == (1000, P * 8)
        p0 = pl[:900, :5].float()
        assert torch.equal(p0, x[:900].to(torch.bfloat16).float())
        assert torch.all(pl[:900, 5:8] == 0)
        if P == 2:
            assert torch.equal(pl[:900, 8:13].float(), (x[:900] - p0).to(torch.bfloat16).float())
        back = ops.from_planes(pl, d_n, P)[:900, :5]
        assert ((back - x[:900]).abs() <= x[:900].abs() * (2.0 ** -8 if P == 1 else 2.0 ** -16)).all()


@pytest.mark.parametrize('subm,cin,cout,B,spare', [(True, 16, 16, 2, 0), (True, 64, 64, 2, 0), (False, 32, 64, 2, 0),
                                                   (True, 32, 32, 5, 300)],
                         ids=['True-16-16', 'True-64-64', 'False-32-64', 'True-32-32-B5-spare300'])
def test_tile_schedule_is_a_bit_exact_permutation(cuda, subm, cin, cout, B, spare):
    """Row-major table == k-major table; dz_rulebook_schedule: `order` is a permutation of the valid rows grouped by
    neighbour-mask digest, a 128-row tile then touches fewer kernel offsets than in coordinate order, the tile launch order
    is heaviest-first with the capacity tiles beyond the count last, and the scheduled tensor-core conv returns
    bit-identical features (same per-row accumulation order), incl. rows beyond the count being left alone.  `spare`:
    capacity rows of a submanifold level beyond its count; the B = 5 case is a batch of more than two frames."""
    from detzero_b200 import ops
    from detzero_b200.spconv.pytorch import SparseConvTensor
    shape = [13, 64, 64]
    idx, f = _sparse_input(cuda, 77, B, shape, 0.05, cin)
    t = SparseConvTensor(f.to(cuda), torch.from_numpy(idx).to(cuda), shape, B)
    if subm:
        n = len(idx)
        cap = out_cap = n + spare
        coords = torch.zeros((cap, 4), dtype=torch.int32, device=cuda)
        coords[:n] = t._idx
        sws = ops.new_sched_ws(cap, cuda)
        (nbr, tab), d_n = ops.rulebook_subm(coords, t._count, cap, t.grid_index(), [3, 3, 3], layout='both', sched_ws=sws), t._count
    else:
        cap = out_cap = len(idx) * 2
        sws = ops.new_sched_ws(cap, cuda)
        oc, d_n, oi, (nbr, tab), odhw = ops.rulebook_conv(t._idx, t._count, t._cap, t.grid_index(), [3, 3, 3], [2, 2, 2], [1, 1, 1],
                                                          out_cap=out_cap, layout='both', sched_ws=sws)
        n = int(d_n.item())
    k_major = nbr[:, :n].cpu().numpy()
    assert np.array_equal(tab[:n, :27].cpu().numpy().T, k_major)
    bits = ((k_major >= 0).astype(np.int64) << np.arange(27)[:, None]).sum(0)
    assert np.array_equal(tab[:n, 27].cpu().numpy().astype(np.int64), bits)
    assert torch.equal(ops.table_to_rows(nbr)[:n], tab[:n])
    order, tab_tiles = ops.rulebook_schedule(tab, d_n, sws, K=27)
    o = order[:n].cpu().numpy()
    assert np.array_equal(np.sort(o), np.arange(n))
    tiles = (cap + 127) // 128
    to = order[cap:cap + tiles].cpu().numpy()                                # tile launch order: a permutation, heaviest tile first
    assert np.array_equal(np.sort(to), np.arange(tiles))

    def tile_work(valid):
        v = np.zeros((27, tiles * 128), bool)
        v[:, :n] = valid
        return v.reshape(27, tiles, 128).any(2).sum(0)
    work = tile_work(k_major[:, o] >= 0)
    assert np.all(np.diff(work[to]) <= 0)
    live = to[to * 128 < n]
    assert np.array_equal(np.sort(live), np.arange((n + 127) // 128)) and np.all(to[len(live):] * 128 >= n)   # empty tiles last
    # tile-major copy of the scheduled table: tile j = 27 neighbour planes + the row plane; tile masks appended to `order`
    tn = (n + 127) // 128
    tt = tab_tiles[:tn].cpu().numpy()
    rows_plane = np.full(tn * 128, -1, np.int64); rows_plane[:n] = o
    assert np.array_equal(tt[:, 27, :].reshape(-1), rows_plane)
    want_planes = np.full((27, tn * 128), -1, np.int64); want_planes[:, :n] = k_major[:, o]
    assert np.array_equal(tt[:, :27, :].transpose(1, 0, 2).reshape(27, -1), want_planes)
    tmask = order[cap + tiles:cap + 2 * tiles].cpu().numpy()[:tn]
    assert np.array_equal(tmask, (((want_planes >= 0).reshape(27, tn, 128).any(2)).astype(np.int64) << np.arange(27)[:, None]).sum(0))
    assert work.sum() <= tile_work(k_major >= 0).sum()
    g = np.random.default_rng(9)
    w = torch.from_numpy(g.normal(0, 0.2, (cout, 3, 3, 3, cin)).astype(np.float32))
    scale = torch.from_numpy(g.uniform(0.5, 1.5, cout).astype(np.float32)).to(cuda)
    shift = torch.from_numpy(g.normal(0, 0.1, cout).astype(np.float32)).to(cuda)
    res = torch.from_numpy(g.normal(0, 1, (out_cap, cout)).astype(np.float32)).to(cuda)
    for mode in (_lib.DZ_TF32, _lib.DZ_TF32X3):
        wp = ops.pack_spconv_weight(w, mode).to(cuda)
        a = ops.spconv_fwd(t._feat, tab, d_n, out_cap, wp, scale, shift, res, True, mode, kshape=(27, cin, cout),
                           out=torch.full((out_cap, cout), -7.0, device=cuda))
        b = ops.spconv_fwd(t._feat, tab, d_n, out_cap, wp, scale, shift, res, True, mode, kshape=(27, cin, cout),
                           out=torch.full((out_cap, cout), -7.0, device=cuda), row_order=order)
        c = ops.spconv_fwd(t._feat, nbr, d_n, out_cap, wp, scale, shift, res, True, mode, kshape=(27, cin, cout),
                           out=torch.full((out_cap, cout), -7.0, device=cuda))      # k-major table converted on the fly
        assert torch.equal(a, b) and torch.equal(a, c), mode
        assert torch.all(a[n:] == -7.0)
    for mode in (_lib.DZ_BF16X2, _lib.DZ_BF16):           # persistent bf16-plane kernel: scheduled == unscheduled, bit for bit
        P = _lib.PLANES[mode]
        wp = ops.pack_spconv_weight(w, mode).to(cuda)
        fp, rp = ops.to_planes(t._feat, t._count, P), ops.to_planes(res, d_n, P)
        fill = lambda: torch.full((out_cap, P * cout), -7.0, device=cuda, dtype=torch.bfloat16)
        a = ops.spconv_fwd(fp, tab, d_n, out_cap, wp, scale, shift, rp, True, mode, kshape=(27, cin, cout), out=fill(), layout='row')
        b = ops.spconv_fwd(fp, tab, d_n, out_cap, wp, scale, shift, rp, True, mode, kshape=(27, cin, cout), out=fill(), row_order=order, layout='row')
        c = ops.spconv_fwd(fp, tab, d_n, out_cap, wp, scale, shift, rp, True, mode, kshape=(27, cin, cout), out=fill(), row_order=order, layout='row',
                           tab_tiles=tab_tiles)                              # fast path: one bulk copy per tile
        assert torch.equal(a, b) and torch.equal(a, c), mode
        assert torch.all(a[n:] == -7.0) and torch.all(c[n:] == -7.0)
    with pytest.raises(RuntimeError):         # the exact-fp32 kernel compacts per offset itself: a schedule is refused loudly
        ops.spconv_fwd(t._feat, nbr, d_n, out_cap, ops.pack_spconv_weight(w, _lib.DZ_F32).to(cuda), scale, shift, res, True,
                       _lib.DZ_F32, kshape=(27, cin, cout), row_order=order)


@pytest.mark.parametrize('kind,mode,tol', [('VoxelBackBone8x', 'fp32', 2e-5), ('VoxelResBackBone8x', 'fp32', 2e-5),
                                           ('VoxelBackBone8x', 'tf32', 5e-3), ('VoxelResBackBone8x', 'tf32', 5e-3),
                                           ('VoxelBackBone8x', 'tf32x3', 2e-4), ('VoxelResBackBone8x', 'tf32x3', 2e-4),
                                           ('VoxelBackBone8x', 'bf16x2', 2e-4), ('VoxelResBackBone8x', 'bf16x2', 2e-4),
                                           ('VoxelBackBone8x', 'bf16', 3e-2), ('VoxelResBackBone8x', 'bf16', 3e-2)])
def test_backbone3d_vs_oracle(cuda, kind, mode, tol):
    from detzero_b200.det import cp_modules
    cfg = util.model_cfg(kind).BACKBONE_3D
    cfg.COMPUTE_MODE = mode
    m = cp_modules[kind](model_cfg=cfg, input_channels=5, grid_size=[192, 192, 40]).eval()
    sd = weights.load_seeded(m, 7)
    m = m.to(cuda)
    clouds = [util.clustered_cloud(25000, 41), util.clustered_cloud(12000, 42)]
    ref = oracle.Point2VoxelCPU3d(util.VOXEL, util.SMALL_RANGE, 5, 5, 40000)
    feats, coords = [], []
    for b, p in enumerate(clouds):
        v, c, n = ref.point_to_voxel(p)
        feats.append(det_ref.mean_vfe(v, n)); coords.append(np.pad(c, ((0, 0), (1, 0)), constant_values=b))
    feats, coords = torch.cat(feats), np.concatenate(coords).astype(np.int32)
    want = det_ref.voxel_backbone(sd, '', feats, coords, m.sparse_shape, 2, res=(kind == 'VoxelResBackBone8x'))
    bd = {'voxel_features': feats.to(cuda), 'voxel_coords': torch.from_numpy(coords).to(cuda), 'batch_size': 2}
    with torch.no_grad():
        bd = m(bd)
    for name, got in list(bd['multi_scale_3d_features'].items()) + [('out', bd['encoded_spconv_tensor'])]:
        w = want[name]
        assert np.array_equal(got.indices.cpu().numpy(), w.idx), name       # same sites, same (sorted) order
        assert got.spatial_shape == w.shape
        assert util.rel_err(got.features.cpu(), w.f) < tol, name


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('cin,cout,k,stride,pad,H,W', [(64, 64, 3, 1, 1, 24, 20), (256, 128, 3, 1, 1, 13, 11),
                                                       (128, 256, 3, 2, 1, 24, 24), (64, 12, 3, 1, 1, 9, 10),
                                                       (128, 256, 1, 1, 0, 12, 12), (384, 12, 3, 1, 1, 8, 8)])
def test_conv2d_fp32(cuda, cin, cout, k, stride, pad, H, W):
    from detzero_b200 import ops
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) * 0.05
    scale, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1
    xh = x.permute(0, 2, 3, 1).contiguous().to(cuda)
    for mode in ('fp32', 'tf32'):
        if mode == 'tf32' and cin % 32:
            continue
        m = _lib.MODES[mode]
        out = ops.conv2d(xh, ops.pack_conv_weight(w, m).to(cuda), (k, k, cin, cout), stride, pad, scale.to(cuda), shift.to(cuda), True,
                         mode=m)
        sa.assert_conv2d(out, xh, w, stride, pad, scale, shift, True, mode, mode)


@pytest.mark.parametrize('cin,cout,H,W,coff,cstride', [(128, 128, 136, 184, 0, 128), (64, 64, 152, 168, 32, 160), (256, 256, 94, 94, 0, 256)])
def test_conv2d_tf32_many_tiles(cuda, cin, cout, H, W, coff, cstride):
    """many 8x16 patches (more than one per SM and cout slice) through the tensor-core conv,
    ragged edges (H, W not multiples of the patch), output written at a channel offset of a wider (concat) tensor through the
    TMA-store epilogue -- the neighbouring channels must stay untouched"""
    from detzero_b200 import ops
    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, cin, H, W, generator=g)
    w = torch.randn(cout, cin, 3, 3, generator=g) * 0.05
    scale, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1
    xh = x.permute(0, 2, 3, 1).contiguous().to(cuda)
    out = torch.full((1, H, W, cstride), -3.0, device=cuda)
    ops.conv2d(xh, ops.pack_conv_weight(w, _lib.DZ_TF32).to(cuda), (3, 3, cin, cout), 1, 1,
               scale.to(cuda), shift.to(cuda), True, out=out, out_coff=coff, mode=_lib.DZ_TF32)
    sa.assert_conv2d(out[..., coff:coff + cout], xh, w, 1, 1, scale, shift, True, 'tf32', 'many tiles')
    assert torch.all(out[..., :coff] == -3.0) and torch.all(out[..., coff + cout:] == -3.0)


@pytest.mark.parametrize('s', [1, 2])
def test_deconv2d_fp32_concat(cuda, s):
    from detzero_b200 import ops
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 64, 7, 9, generator=g)
    w = torch.randn(64, 32, s, s, generator=g) * 0.1
    xh = x.permute(0, 2, 3, 1).contiguous().to(cuda)
    for mode in ('fp32', 'tf32'):
        out = torch.zeros(2, 7 * s, 9 * s, 48, device=cuda)
        ops.deconv2d(xh, ops.pack_deconv_weight(w, _lib.MODES[mode]).to(cuda), (s, 64, 32), None, None,
                     False, out=out, out_coff=16, mode=_lib.MODES[mode])
        sa.assert_conv2d(out[..., 16:], xh, w, 1, 0, None, None, False, mode, mode, transposed=True)
        assert out[..., :16].abs().max().item() == 0


@pytest.mark.parametrize('B,cin,cout,H,W,coff,ctot', [(3, 256, 256, 94, 94, 256, 512), (3, 64, 64, 10, 21, 0, 64), (2, 128, 96, 30, 17, 32, 160)])
def test_deconv2d_tf32_strided_tma_store(cuda, B, cin, cout, H, W, coff, ctot):
    """ConvTranspose2d(kernel = stride = 2) on the tensor-core path with an even Ho: the epilogue stores through the 5-D
    [C][dx][x][dy][b*Ho + y] view of the NHWC output (rows past Ho of the last tile are skipped, not wrapped into the next frame;
    pixels past Wo are clipped), into a channel slice of a wider (concatenated) tensor"""
    from detzero_b200 import ops
    g = torch.Generator().manual_seed(B + H)
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cin, cout, 2, 2, generator=g) * 0.05
    scale, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1
    xh = x.permute(0, 2, 3, 1).contiguous().to(cuda)
    out = torch.full((B, 2 * H, 2 * W, ctot), -3.0, device=cuda)
    ops.deconv2d(xh, ops.pack_deconv_weight(w, _lib.DZ_TF32).to(cuda), (2, cin, cout), scale.to(cuda),
                 shift.to(cuda), True, out=out, out_coff=coff, mode=_lib.DZ_TF32)
    sa.assert_conv2d(out[..., coff:coff + cout], xh, w, 1, 0, scale, shift, True, 'tf32', 'strided store', transposed=True)
    assert torch.all(out[..., :coff] == -3.0) and torch.all(out[..., coff + cout:] == -3.0)


def test_sparse_to_bev(cuda):
    from detzero_b200.spconv.pytorch import SparseConvTensor
    shape, B = [2, 24, 24], 2
    idx, f = _sparse_input(cuda, 51, B, shape, 0.2, 128)
    t = SparseConvTensor(f.to(cuda), torch.from_numpy(idx).to(cuda), shape, B)
    ref = spconv_ref.dense_from_sparse(f, idx, shape, B)
    assert torch.equal(t.dense().cpu(), ref)


def _dense_models(cuda, seed=9):
    from detzero_b200.det import cp_modules
    cfg = util.model_cfg()
    b2d = cp_modules['BaseBEVBackbone'](model_cfg=cfg.BACKBONE_2D, input_channels=256).eval()
    head = cp_modules['CenterHead'](model_cfg=cfg.DENSE_HEAD, input_channels=512, num_class=3, class_names=util.CLASS_NAMES,
                                    grid_size=[192, 192, 40], point_cloud_range=util.SMALL_RANGE, voxel_size=util.VOXEL).eval()
    sd2, sdh = weights.load_seeded(b2d, seed), weights.load_seeded(head, seed + 1)
    return cfg, b2d.to(cuda), head.to(cuda), sd2, sdh


def test_bev_backbone_and_head_maps(cuda):
    cfg, b2d, head, sd2, sdh = _dense_models(cuda)
    x = torch.randn(2, 256, 24, 24, generator=torch.Generator().manual_seed(1))
    ref2d = det_ref.bev_backbone(sd2, '', x, [5, 5], [1, 2], [1, 2])
    names = ['center', 'center_z', 'dim', 'rot', 'iou', 'hm']
    refmaps = det_ref.center_head_maps(sdh, '', ref2d, names)
    with torch.no_grad():
        bd = b2d({'spatial_features': x.to(cuda)})
        assert bd['spatial_features_2d'].shape == ref2d.shape
        assert util.rel_err(bd['spatial_features_2d'].cpu(), ref2d) < 2e-5
        bd['batch_size'] = 2
        bd = head(bd)
    for n in names:
        assert util.rel_err(head.forward_ret_dict['pred_dicts'][0][n].cpu(), refmaps[n]) < 5e-5, n


def test_iou_and_nms(cuda):
    from detzero_b200 import ops
    g = np.random.default_rng(2)
    n = 300
    boxes = np.concatenate([g.uniform(-20, 20, (n, 2)), g.uniform(-1, 1, (n, 1)), g.uniform(1.5, 5, (n, 2)),
                            g.uniform(1, 2, (n, 1)), g.uniform(-3.2, 3.2, (n, 1))], axis=1).astype(np.float32)
    boxes[100:200, :2] = boxes[:100, :2] + g.normal(0, 0.3, (100, 2)).astype(np.float32)     # overlapping clusters
    boxes[100:200, 3:7] = boxes[:100, 3:7] + g.normal(0, 0.05, (100, 4)).astype(np.float32)
    iou_ref = oracle.boxes_iou_bev(boxes, boxes)
    iou = ops.boxes_iou_bev(torch.from_numpy(boxes).to(cuda), torch.from_numpy(boxes).to(cuda)).cpu().numpy()
    assert np.abs(iou - iou_ref).max() < 1e-4
    scores = np.sort(g.uniform(0.05, 1, n).astype(np.float32))[::-1].copy()
    keep_ref = oracle.nms_bev_sorted(boxes, 0.7)
    margin = np.abs(iou_ref - 0.7)
    assert margin[np.triu_indices(n, 1)].min() > 1e-4, 'test boxes too close to the threshold'
    cap = 512
    pb = np.zeros((1, cap, 7), np.float32); pb[0, :n] = boxes
    ps = np.zeros((1, cap), np.float32); ps[0, :n] = scores
    out, d_out = ops.nms_bev(torch.from_numpy(pb).to(cuda), torch.from_numpy(ps).to(cuda),
                             torch.zeros((1, cap), dtype=torch.int32, device=cuda),
                             torch.tensor([n], dtype=torch.int32, device=cuda), 0.7, 500, label_offset=1)
    k = int(d_out.item())
    assert k == len(keep_ref)
    assert np.array_equal(out[0, :k, :7].cpu().numpy(), boxes[keep_ref])
    assert np.array_equal(out[0, :k, 7].cpu().numpy(), scores[keep_ref])
    assert out[0, k:].abs().max().item() == 0


@pytest.mark.parametrize('H,W', [(24, 24), (96, 80)])      # 96x80: > 4096 scores above the threshold -> full-map select path
def test_decode_and_nms_vs_oracle(cuda, H, W):
    from detzero_b200 import ops
    g = torch.Generator().manual_seed(12)
    B = 2
    maps = {'center': torch.rand(B, 2, H, W, generator=g), 'center_z': torch.randn(B, 1, H, W, generator=g),
            'dim': torch.randn(B, 3, H, W, generator=g) * 0.3 + 0.8, 'rot': torch.randn(B, 2, H, W, generator=g),
            'iou': torch.rand(B, 1, H, W, generator=g) * 1.4 - 0.2, 'hm': torch.randn(B, 3, H, W, generator=g) * 2 - 1}
    post = dict(MAX_OBJ_PER_SAMPLE=500, SCORE_THRESH=0.03, POST_CENTER_LIMIT_RANGE=[-80, -80, -10.0, 80, 80, 10.0],
                NMS_THRESH=0.7, NMS_PRE_MAXSIZE=4096, NMS_POST_MAXSIZE=500)
    want = det_ref.generate_predicted_boxes(maps, util.SMALL_RANGE, util.VOXEL, 8, post, use_iou=True)
    order = ['center', 'center_z', 'dim', 'rot', 'iou', 'hm']
    hm = torch.cat([maps[k] for k in order], dim=1).permute(0, 2, 3, 1).contiguous().to(cuda)
    layout, off = {}, 0
    for k in order:
        layout[k] = off; off += maps[k].shape[1]
    boxes, scores, labels, d_n = ops.centerhead_decode(hm, layout, 3, 500, util.SMALL_RANGE, util.VOXEL, 8,
                                                       post['POST_CENTER_LIMIT_RANGE'], 0.03, True)
    out, d_out = ops.nms_bev(boxes, scores, labels, d_n, 0.7, 500, label_offset=1)
    for b in range(B):
        k = int(d_out[b].item())
        assert k == want[b]['pred_boxes'].shape[0]
        assert (out[b, :k, :7].cpu() - want[b]['pred_boxes']).abs().max().item() < 1e-3       # metres / radians
        assert (out[b, :k, 7].cpu() - want[b]['pred_scores']).abs().max().item() < 1e-6
        assert torch.equal(out[b, :k, 8].cpu().long(), want[b]['pred_labels'])


def test_centerpoint_end_to_end(cuda):
    """raw points -> final boxes through the registry-built CenterPoint vs the CPU oracle chain"""
    from detzero_b200.det import build_network, load_data_to_gpu
    from detzero_b200.det.dataset import SyntheticWaymoDataset, default_waymo_1sweep_cfg
    dcfg = default_waymo_1sweep_cfg()
    dcfg.POINT_CLOUD_RANGE = util.SMALL_RANGE
    ds = SyntheticWaymoDataset(dcfg, util.CLASS_NAMES, training=False, num_frames=2, n_points=30000)
    cfg = util.model_cfg('VoxelResBackBone8x')
    model = build_network(cfg, 3, ds).eval()
    sd = weights.load_seeded(model, 21)
    model = model.to(cuda)
    clouds = [util.clustered_cloud(30000, 61, c=6), util.clustered_cloud(20000, 62, c=6)]
    items = []
    for i, p in enumerate(clouds):
        d = {'points': p, 'frame_id': str(i)}
        items.append(ds.data_processor.forward(ds.point_feature_encoder.forward(d)))
    batch = ds.collate_batch(items)
    load_data_to_gpu(batch, cuda)
    with torch.no_grad():
        pred_dicts, _ = model(batch)
    # oracle chain
    vox = oracle.Point2VoxelCPU3d(util.VOXEL, util.SMALL_RANGE, 5, 5, 200000)
    feats, coords = [], []
    for b, d in enumerate(items):
        v, c, n = vox.point_to_voxel(d['points'])
        feats.append(det_ref.mean_vfe(v, n)); coords.append(np.pad(c, ((0, 0), (1, 0)), constant_values=b))
    lv = det_ref.voxel_backbone(sd, 'backbone3d.', torch.cat(feats), np.concatenate(coords), [41, 192, 192], 2, res=True)
    sf = det_ref.height_compression(lv['out'])
    s2d = det_ref.bev_backbone(sd, 'backbone2d.', sf, [5, 5], [1, 2], [1, 2])
    maps = det_ref.center_head_maps(sd, 'dense_head.', s2d, ['center', 'center_z', 'dim', 'rot', 'iou', 'hm'])
    post = dict(MAX_OBJ_PER_SAMPLE=500, SCORE_THRESH=0.03, POST_CENTER_LIMIT_RANGE=[-80, -80, -10.0, 80, 80, 10.0],
                NMS_THRESH=0.7, NMS_PRE_MAXSIZE=4096, NMS_POST_MAXSIZE=500)
    want = det_ref.generate_predicted_boxes(maps, util.SMALL_RANGE, util.VOXEL, 8, post, use_iou=True)
    assert util.rel_err(batch['spatial_features_2d'].cpu(), s2d) < 1e-4
    for b in range(2):
        _assert_same_detections(pred_dicts[b], want[b])


def _assert_same_detections(got, want, score_tol=1e-5, box_tol=1e-3, count_slack=0):
    """same detections up to the order of (near-)tied scores: counts equal (up to `count_slack` boxes that sit on the score /
    NMS thresholds in the reduced-precision modes), sorted scores equal, every oracle box has a product box within box_tol
    m / rad (+1e-4 relative: exp() of the size regressions)"""
    ng, nw = got['pred_boxes'].shape[0], want['pred_boxes'].shape[0]
    assert abs(ng - nw) <= count_slack, (ng, nw)
    gs, ws = got['pred_scores'].cpu().sort(descending=True)[0], want['pred_scores'].sort(descending=True)[0]
    if count_slack == 0:
        assert (gs - ws).abs().max().item() < score_tol
    # the label is part of the match: one BEV cell can fire for two classes with the very same box
    gb = torch.cat([got['pred_boxes'].cpu().double(), got['pred_scores'].cpu().double()[:, None] * (box_tol / score_tol),
                    got['pred_labels'].cpu().double()[:, None]], dim=1)
    wb = torch.cat([want['pred_boxes'].double(), want['pred_scores'].double()[:, None] * (box_tol / score_tol),
                    want['pred_labels'].double()[:, None]], dim=1)
    scale = 1.0 + 0.1 * wb[:, None, :].abs()
    scale[..., 7] = 1.0                                     # the (rescaled) score is compared absolutely
    diff = (gb[None, :, :] - wb[:, None, :]).abs() / scale
    nearest = diff.max(dim=2)[0].min(dim=1)[0]
    bad = int((nearest >= box_tol).sum().item())
    assert bad <= count_slack, (bad, nearest.max().item())


def test_dynamic_vfe_into_backbone(cuda):
    """BASELINE configs[2] path (multi-sweep): DynamicMeanVFE (key order b,x,y,z) -> VoxelResBackBone8x; the backbone builds
    its grid index from the arbitrary-order coordinate list"""
    from detzero_b200.det import cp_modules
    cfg = util.model_cfg('VoxelResBackBone8x')
    grid = [192, 192, 40]
    vfe = cp_modules['DynamicMeanVFE'](model_cfg=cfg.VFE, num_point_features=6, voxel_size=util.VOXEL, grid_size=grid,
                                       point_cloud_range=util.SMALL_RANGE)
    bb = cp_modules['VoxelResBackBone8x'](model_cfg=cfg.BACKBONE_3D, input_channels=6, grid_size=grid).eval()
    sd = weights.load_seeded(bb, 17)
    bb = bb.to(cuda)
    clouds = [util.clustered_cloud(30000, 71, c=6), util.clustered_cloud(18000, 72, c=6)]
    pts = np.concatenate([np.pad(p, ((0, 0), (1, 0)), constant_values=b) for b, p in enumerate(clouds)]).astype(np.float32)
    mean_ref, coords_ref = det_ref.dynamic_mean_vfe(pts, util.SMALL_RANGE, util.VOXEL, grid)
    want = det_ref.voxel_backbone(sd, '', mean_ref, coords_ref.numpy(), bb.sparse_shape, 2, res=True)
    def attempt():
        bd = {'points': torch.from_numpy(pts).to(cuda), 'batch_size': 2}
        with torch.no_grad():
            bd = bb(vfe(bd))
        m = int(bd['voxel_count'].item())
        got = bd['encoded_spconv_tensor']
        checks = {'voxel count': m == coords_ref.shape[0],
                  'voxel coords': m == coords_ref.shape[0] and torch.equal(bd['voxel_coords'][:m].cpu(), coords_ref),
                  'output sites': np.array_equal(got.indices.cpu().numpy(), want['out'].idx)}
        checks['output features'] = checks['output sites'] and util.rel_err(got.features.cpu(), want['out'].f) < 1e-4
        return [k for k, ok in checks.items() if not ok]

    # round 1 saw an intermittent failure here: id()-keyed global caches of folded BN / packed weights handed a freed model's
    # tensors to the next model; the caches now live on the modules.  No retry, no xfail.
    failed = attempt()
    assert not failed, failed


def test_centerpoint_end_to_end_tf32(cuda):
    """the default tensor-core configuration (TF32 sparse + dense convs): same detections as the fp32 oracle chain within
    5 cm / 0.05 rad / 0.02 score for at least 90 % of the boxes (TF32 perturbs scores near the NMS / score thresholds)"""
    from detzero_b200.det import build_network, load_data_to_gpu
    from detzero_b200.det.dataset import SyntheticWaymoDataset, default_waymo_1sweep_cfg
    dcfg = default_waymo_1sweep_cfg()
    dcfg.POINT_CLOUD_RANGE = util.SMALL_RANGE
    ds = SyntheticWaymoDataset(dcfg, util.CLASS_NAMES, training=False, num_frames=1, n_points=30000)
    outs = {}
    clouds = [util.clustered_cloud(30000, 61, c=6)]
    for mode in ('fp32', 'tf32'):
        cfg = util.model_cfg('VoxelBackBone8x', mode)
        model = build_network(cfg, 3, ds).eval()
        weights.load_seeded(model, 21)
        model = model.to(cuda)
        items = [ds.data_processor.forward(ds.point_feature_encoder.forward({'points': p.copy(), 'frame_id': '0'})) for p in clouds]
        batch = load_data_to_gpu(ds.collate_batch(items), cuda)
        with torch.no_grad():
            outs[mode] = model(batch)[0][0]
    a, b = outs['fp32'], outs['tf32']
    assert abs(a['pred_boxes'].shape[0] - b['pred_boxes'].shape[0]) <= max(3, a['pred_boxes'].shape[0] // 20)
    if a['pred_boxes'].shape[0]:
        ga = torch.cat([a['pred_boxes'][:, :3], a['pred_boxes'][:, 6:7], a['pred_scores'][:, None] * 2.5, a['pred_labels'][:, None].float()], 1)
        gb = torch.cat([b['pred_boxes'][:, :3], b['pred_boxes'][:, 6:7], b['pred_scores'][:, None] * 2.5, b['pred_labels'][:, None].float()], 1)
        d = (ga[:, None, :] - gb[None, :, :]).abs().max(dim=2)[0].min(dim=1)[0]
        assert (d < 0.05).float().mean().item() >= 0.9


def test_tile_schedule_edge_cases(cuda):
    """empty level (count 0), a level smaller than one tile, and the K = 3 (3,1,1)/(2,1,1) rulebook of conv_out: the schedule
    stays a permutation, and scheduled == unscheduled bit for bit (nothing written for a count of 0)"""
    from detzero_b200 import ops
    from detzero_b200.spconv.pytorch import SparseConvTensor
    shape, B = [9, 24, 24], 1
    idx, f = _sparse_input(cuda, 5, B, shape, 0.06, 64)
    t = SparseConvTensor(f.to(cuda), torch.from_numpy(idx).to(cuda), shape, B)
    cap = len(idx)
    g = np.random.default_rng(3)
    w27 = ops.pack_spconv_weight(torch.from_numpy(g.normal(0, 0.2, (64, 3, 3, 3, 64)).astype(np.float32)), _lib.DZ_TF32).to(cuda)
    for n_fake in (0, 5):
        d_n = torch.tensor([n_fake], dtype=torch.int32, device=cuda)
        sws = ops.new_sched_ws(cap, cuda)
        tab = ops.rulebook_subm(t._idx, d_n, cap, t.grid_index(), [3, 3, 3], layout='row', sched_ws=sws)
        order = ops.rulebook_schedule(tab, d_n, sws)
        assert np.array_equal(np.sort(order[:n_fake].cpu().numpy()), np.arange(n_fake))
        tiles = (cap + 127) // 128
        assert np.array_equal(np.sort(order[cap:cap + tiles].cpu().numpy()), np.arange(tiles))
        a = ops.spconv_fwd(t._feat, tab, d_n, cap, w27, None, None, None, True, _lib.DZ_TF32, kshape=(27, 64, 64),
                           out=torch.full((cap, 64), -7.0, device=cuda))
        b = ops.spconv_fwd(t._feat, tab, d_n, cap, w27, None, None, None, True, _lib.DZ_TF32, kshape=(27, 64, 64),
                           out=torch.full((cap, 64), -7.0, device=cuda), row_order=order)
        assert torch.equal(a, b) and torch.all(a[n_fake:] == -7.0)
    # conv_out geometry: kernel (3,1,1), stride (2,1,1), no padding -> K = 3
    out_cap = 2 * cap
    sws = ops.new_sched_ws(out_cap, cuda)
    oc, d_n, oi, (nbr, tab), odhw = ops.rulebook_conv(t._idx, t._count, t._cap, t.grid_index(), [3, 1, 1], [2, 1, 1], [0, 0, 0],
                                                      out_cap=out_cap, layout='both', sched_ws=sws)
    n = int(d_n.item())
    assert 0 < n <= out_cap
    assert np.array_equal(tab[:n, :3].cpu().numpy().T, nbr[:, :n].cpu().numpy()) and torch.all(tab[:n, 3:27] == -1)
    order = ops.rulebook_schedule(tab, d_n, sws)
    assert np.array_equal(np.sort(order[:n].cpu().numpy()), np.arange(n))
    w3 = ops.pack_spconv_weight(torch.from_numpy(g.normal(0, 0.2, (128, 3, 1, 1, 64)).astype(np.float32)), _lib.DZ_TF32).to(cuda)
    a = ops.spconv_fwd(t._feat, tab, d_n, out_cap, w3, None, None, None, True, _lib.DZ_TF32, kshape=(3, 64, 128))
    b = ops.spconv_fwd(t._feat, tab, d_n, out_cap, w3, None, None, None, True, _lib.DZ_TF32, kshape=(3, 64, 128), row_order=order)
    assert torch.equal(a[:n], b[:n])


def test_batched_frames_equal_single_frames(cuda):
    """a batch of two frames through the default tensor-core detector gives, frame by frame, exactly the detections of the two
    single-frame runs (tiles mix rows of both frames, but every row's arithmetic is unchanged)"""
    from detzero_b200.det import build_network, load_data_to_gpu
    from detzero_b200.det.dataset import SyntheticWaymoDataset, default_waymo_1sweep_cfg
    dcfg = default_waymo_1sweep_cfg()
    dcfg.POINT_CLOUD_RANGE = util.SMALL_RANGE
    ds = SyntheticWaymoDataset(dcfg, util.CLASS_NAMES, training=False, num_frames=2, n_points=30000)
    model = build_network(util.model_cfg('VoxelBackBone8x', 'tf32'), 3, ds).eval()
    weights.load_seeded(model, 21)
    model = model.to(cuda)
    clouds = [util.clustered_cloud(30000, 61, c=6), util.clustered_cloud(22000, 62, c=6)]
    items = [ds.data_processor.forward(ds.point_feature_encoder.forward({'points': p.copy(), 'frame_id': str(k)})) for k, p in enumerate(clouds)]
    with torch.no_grad():
        both = model(load_data_to_gpu(ds.collate_batch(items), cuda))[0]
        singles = [model(load_data_to_gpu(ds.collate_batch([it]), cuda))[0][0] for it in items]
    assert sum(s['pred_boxes'].shape[0] for s in singles) > 0
    for k in range(2):
        for key in ('pred_boxes', 'pred_scores', 'pred_labels'):
            assert torch.equal(both[k][key], singles[k][key]), (k, key)


@pytest.mark.parametrize('cin,cout,k,stride,pad,H,W,B,coff,cstride', [(128, 128, 3, 1, 1, 188, 188, 2, 0, 128), (256, 256, 3, 1, 1, 94, 94, 8, 0, 256),
                                                                      (128, 256, 3, 2, 1, 187, 189, 4, 0, 256), (256, 128, 3, 1, 1, 100, 84, 4, 64, 256),
                                                                      (128, 256, 1, 1, 0, 150, 150, 2, 256, 512),
                                                                      # 3x3 stride-1 at every tile width: 64 (shared conv), 32 with a ragged Cout
                                                                      # (fused head stage 2), 3 x 128 (fused head stage 1), ragged image edges
                                                                      (512, 64, 3, 1, 1, 188, 188, 2, 0, 64), (384, 12, 3, 1, 1, 100, 90, 4, 0, 12),
                                                                      (64, 384, 3, 1, 1, 95, 93, 4, 0, 384), (128, 128, 3, 1, 1, 61, 67, 8, 128, 384)])
def test_conv2d_tf32_halo_and_generic_kernels(cuda, cin, cout, k, stride, pad, H, W, B, coff, cstride):
    """the BEV-backbone and head shapes at batch sizes that give several tiles per SM: Cout = 256 (two 128-wide weight tiles per
    patch), odd tile counts, ragged edges, stride 2, 1x1, channel-offset (concat) output; the 3x3 stride-1 shapes run through the
    HALO variant (one (16+2) x (8+2) activation tile per 32-channel slice, nine shifted wgmma descriptors) at every tile width"""
    from detzero_b200 import ops
    g = torch.Generator().manual_seed(13)
    x = torch.randn(B, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) * 0.05
    scale, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    xh = x.permute(0, 2, 3, 1).contiguous().to(cuda)
    out = torch.full((B, Ho, Wo, cstride), -3.0, device=cuda)
    ops.conv2d(xh, ops.pack_conv_weight(w, _lib.DZ_TF32).to(cuda), (k, k, cin, cout), stride, pad,
               scale.to(cuda), shift.to(cuda), True, out=out, out_coff=coff, mode=_lib.DZ_TF32)
    sa.assert_conv2d(out[..., coff:coff + cout], xh, w, stride, pad, scale, shift, True, 'tf32', 'conv2d')
    assert torch.all(out[..., :coff] == -3.0) and torch.all(out[..., coff + cout:] == -3.0)

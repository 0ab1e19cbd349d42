"""Element-wise checks of the sparse-conv kernels -- k_spconv_f32 (fp32, its dgrad and SparseInverseConv3d), k_spconv_tf32 (tf32,
tf32x3), k_spconv_bf16 (bf16x2, bf16) and k_spconv_wgrad -- against float64, in every compute mode and every (cin_pad, cout)
instantiation.  The arithmetic contract of each mode and the bounds are in tests/spconv_arith.py (checked on the CPU by
tests/test_spconv_bounds.py).

a. exact operands: the result cannot depend on how the tensor core adds, so every mode must reproduce its contract to the bit,
   on tables built to reach the kernels' edges, unscheduled and scheduled, into sentinel-filled buffers;
b. the operands of every spconv_fwd call of a VoxelBackBone8x and a VoxelResBackBone8x eval forward on two 180 K-point frames,
   against float64 x . w on neighbour pairs restated here from the site coordinates, within bounds derived from operand rounding;
c. the TF32 backbone input is RN-rounded before the first TF32 layer reads it;
d. dgrad, wgrad and SparseInverseConv3d, bit-exact on exact operands and bounded on the real level-1 / level-2 tables."""
import inspect

import numpy as np
import pytest
import torch

from detzero_b200 import _lib, ops
from tests import spconv_arith as sa
from tests.util import assert_within

pytestmark = pytest.mark.gpu
F64 = torch.float64
INST = [(5, 16), (16, 16), (16, 32), (32, 32), (32, 64), (64, 64), (64, 128), (128, 128)]
CAP = 4 * 128 + 37               # four whole 128-row tiles and a partial one
N_IN = 300
SPARE = 40
SENTINEL = {'f32': -7.25e30, 'bf16': -7.0}


def _mode_id(mode):
    return _lib.MODES[mode]


def _cin_pad(cin):
    return 8 if cin <= 8 else cin


def _with_mask(tab, K):
    tab[:, K:] = -1
    tab[:, 27] = ((tab[:, :K] >= 0).to(torch.int64) << torch.arange(K)).sum(1).to(torch.int32)
    tab[:, 28:] = 0
    return tab


def _edge_table(g, K):
    """row-major (CAP, 32) table: tile 0 random; tile 1 without any live offset (the nb == 0 epilogue); tile 2 rows whose only
    neighbour is offset K-1 (a partial last reduction block for cin_pad 8 / 16 / 32), only offset 0, every offset on one input row
    (gathered by many outputs), random; the rest sparse.  Indices are -1 or < N_IN"""
    tab = torch.randint(0, N_IN, (CAP, 32), generator=g, dtype=torch.int32)
    keep = torch.rand(CAP, 32, generator=g)
    tab = torch.where(keep < 0.5, tab, torch.full_like(tab, -1))
    tab[384:] = torch.where(keep[384:] < 0.3, tab[384:], torch.full_like(tab[384:], -1))
    tab[128:256] = -1
    t2 = tab[256:384]
    t2[0::4] = -1
    t2[0::4, K - 1] = torch.randint(0, N_IN, (32,), generator=g, dtype=torch.int32)
    t2[1::4] = -1
    t2[1::4, 0] = torch.randint(0, N_IN, (32,), generator=g, dtype=torch.int32)
    t2[2::4] = 17
    return _with_mask(tab, K)


def _schedule(tab, n, K, g):
    """a valid tile schedule for the first n rows (random row order and tile order) in the layout of dz_rulebook_schedule:
    order = row order (cap) | tile launch order (tiles) | OR of each tile's row masks (tiles), and the tile-major table"""
    cap = tab.shape[0]
    tiles = -(-cap // 128)
    tiles_n = -(-n // 128)
    rows = torch.full((tiles * 128,), -1, dtype=torch.int64)
    rows[:n] = torch.randperm(n, generator=g)
    order = torch.arange(cap, dtype=torch.int32)
    order[:n] = rows[:n].int()
    tile_order = torch.cat([torch.randperm(tiles_n, generator=g), torch.arange(tiles_n, tiles)]).int()
    m = torch.where(rows >= 0, tab[rows.clamp_min(0), 27].long(), torch.zeros_like(rows)).view(tiles, 128)
    masks = torch.from_numpy(np.bitwise_or.reduce(m.numpy(), axis=1)).int()
    tt = torch.where((rows >= 0)[:, None], tab[rows.clamp_min(0), :K], torch.full((tiles * 128, K), -1, dtype=torch.int32))
    tab_tiles = torch.cat([tt, rows.int()[:, None]], 1).view(tiles, 128, K + 1).permute(0, 2, 1).contiguous()
    return torch.cat([order, tile_order, masks]), tab_tiles


def _assert_values(got, want, what):
    """the same values (float64 comparison: -0.0 == 0.0), first difference reported"""
    bad = got.to(F64) != want.to(F64)
    if bool(bad.any()):
        i = np.unravel_index(int(bad.to(torch.uint8).argmax()), tuple(got.shape))
        raise AssertionError('%s: %d differences, first at %s (got %r, contract %r)' % (what, int(bad.sum()), i, got[i].item(),
                                                                                        want[i].item()))


def _run_exact(cuda, mode, cin, cout, K, residual, relu, seed):
    g = torch.Generator().manual_seed(seed)
    mid = _mode_id(mode)
    tab = _edge_table(g, K)
    x, w, scale, shift, res = sa.exact_operands(g, mode, N_IN, cin, cout, K, CAP)
    if not residual:
        res = None
    # the contract, exactly (asserted float32-representable)
    y64 = sa.contract64(mode, tab[:, :K].t(), x, w)
    o64 = sa.epilogue_exact(mode, y64, scale, shift, res, relu)
    assert torch.equal(o64, o64.float().to(F64)), 'exact-operand design broken'
    assert not torch.equal(y64, sa.conv64(tab[:, :K].t(), x, w)) or not sa.dropped(mode, x, w)
    want = sa.output_bits(mode, o64.float())
    # kernel operands
    wp = ops.pack_spconv_weight(w.permute(2, 0, 1).contiguous(), mid).to(cuda)
    P = sa.PLANES.get(mode, 0)
    if P:
        feats = ops.to_planes(x.to(cuda), None, P, _cin_pad(cin))
        rp = None if res is None else ops.to_planes(res.to(cuda), None, P)
        width, dtype, sentinel = P * cout, torch.bfloat16, SENTINEL['bf16']
    else:
        feats, rp = x.to(cuda), (None if res is None else res.to(cuda))
        width, dtype, sentinel = cout, torch.float32, SENTINEL['f32']
    nbr = tab[:, :K].t().contiguous().to(cuda) if mode == 'fp32' else tab.to(cuda)
    sc, sh = scale.to(cuda), shift.to(cuda)
    for n in (0, 1, 127, 129, CAP - 1, CAP + 100):
        d_n = torch.tensor([n], dtype=torch.int32, device=cuda)
        m = min(n, CAP)
        variants = [{}]
        if mode != 'fp32':
            order, tab_tiles = _schedule(tab, m, K, g)
            variants.append({'row_order': order.to(cuda)})
            if P:
                variants.append({'row_order': order.to(cuda), 'tab_tiles': tab_tiles.to(cuda)})
        for kw in variants:
            buf = torch.full((CAP + SPARE, width), sentinel, dtype=dtype, device=cuda)
            ops.spconv_fwd(feats, nbr, d_n, CAP, wp, sc, sh, rp, relu, mid, out=buf[:CAP], kshape=(K, cin, cout),
                           layout='k' if mode == 'fp32' else 'row', **kw)
            what = '%s K=%d (%d, %d) res=%d relu=%d n=%d %s' % (mode, K, cin, cout, residual, relu, n, sorted(kw))
            got = buf.cpu()
            _assert_values(got[:m], want[:m], what)
            assert bool((got[m:] == sentinel).all()), what + ': rows past the count were written'


@pytest.mark.parametrize('mode', sa.MODES)
@pytest.mark.parametrize('cin,cout', INST, ids=['%dx%d' % c for c in INST])
def test_exact_operands_bit_exact(cuda, mode, cin, cout):
    """every mode, every instantiation, K = 27 with and without residual and ReLU (negative power-of-two scales among them), and
    K = 3 where Cout = 128"""
    _run_exact(cuda, mode, cin, cout, 27, False, False, seed=cin * 131 + cout)
    _run_exact(cuda, mode, cin, cout, 27, True, True, seed=cin * 131 + cout + 1)
    if cout == 128:
        _run_exact(cuda, mode, cin, cout, 3, False, True, seed=cin * 131 + cout + 2)
        _run_exact(cuda, mode, cin, cout, 3, True, False, seed=cin * 131 + cout + 3)


# ---------------------------------------------------------------------------------------------------------------------------------
# neighbour pairs restated from the site coordinates (sorted linear keys + searchsorted), independent of the rulebook kernels
# ---------------------------------------------------------------------------------------------------------------------------------
def _keys(idx, shape):
    idx = idx.long()
    return ((idx[:, 0] * shape[0] + idx[:, 1]) * shape[1] + idx[:, 2]) * shape[2] + idx[:, 3]


def _lookup(sites, shape, q):
    """row of each query site q (n, 4) among `sites`, -1 if absent or outside the lattice"""
    keys = _keys(sites, shape)
    sk, perm = torch.sort(keys)
    inside = torch.ones(q.shape[0], dtype=torch.bool, device=q.device)
    for d in range(3):
        inside &= (q[:, d + 1] >= 0) & (q[:, d + 1] < shape[d])
    qk = _keys(q, shape)
    pos = torch.searchsorted(sk, qk).clamp_max(max(sk.numel() - 1, 0))
    hit = inside & (sk[pos] == qk) if sk.numel() else torch.zeros_like(inside)
    return torch.where(hit, perm[pos], torch.full_like(pos, -1))


def _offsets(ks):
    return [(kz, ky, kx) for kz in range(ks[0]) for ky in range(ks[1]) for kx in range(ks[2])]


def pairs_table(in_sites, in_shape, ks, stride, pad, subm, out_sites=None):
    """k-major (K, n_out) table of input rows; for a strided conv also the output site list (sorted by (b, z, y, x))"""
    in_sites = in_sites.long()
    if subm:
        out_sites = in_sites
        tab = [_lookup(in_sites, in_shape, in_sites + torch.tensor([0, kz - ks[0] // 2, ky - ks[1] // 2, kx - ks[2] // 2],
                                                                    device=in_sites.device)) for kz, ky, kx in _offsets(ks)]
        return torch.stack(tab), out_sites, in_shape
    out_shape = [(in_shape[d] + 2 * pad[d] - (ks[d] - 1) - 1) // stride[d] + 1 for d in range(3)]
    cand = []
    for kk in _offsets(ks):
        o = in_sites.clone()
        ok = torch.ones(in_sites.shape[0], dtype=torch.bool, device=in_sites.device)
        for d in range(3):
            num = in_sites[:, d + 1] + pad[d] - kk[d]
            ok &= (num >= 0) & (num % stride[d] == 0) & (num // stride[d] < out_shape[d])
            o[:, d + 1] = num // stride[d]
        cand.append(o[ok])
    ck = torch.unique(_keys(torch.cat(cand), out_shape))
    r = ck.clone()
    sites = torch.zeros(ck.numel(), 4, dtype=torch.long, device=ck.device)
    for d in (3, 2, 1):
        sites[:, d] = r % out_shape[d - 1]
        r //= out_shape[d - 1]
    sites[:, 0] = r
    tab = []
    for kk in _offsets(ks):
        q = sites.clone()
        for d in range(3):
            q[:, d + 1] = sites[:, d + 1] * stride[d] - pad[d] + kk[d]
        tab.append(_lookup(in_sites, in_shape, q))
    return torch.stack(tab), sites, out_shape


# ---------------------------------------------------------------------------------------------------------------------------------
# b. real operands: every spconv_fwd call of two backbone forwards
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def voxels():
    """two config-2 frames (bench.build_inputs: 180 K-point SyntheticWaymoDataset clouds) through the oracle's mean VFE"""
    import bench
    import oracle
    from oracle import det_ref
    from tests import util
    _, batches = bench.build_inputs(1, num_batches=2)
    vox = oracle.Point2VoxelCPU3d(util.VOXEL, util.WAYMO_RANGE, 5, 5, 200000)
    feats, coords = [], []
    for b, batch in enumerate(batches):
        pts = batch['points'][:, 1:]
        v, c, n = vox.point_to_voxel(pts)
        feats.append(torch.as_tensor(np.asarray(det_ref.mean_vfe(v, n)), dtype=torch.float32))
        coords.append(torch.from_numpy(np.pad(c, ((0, 0), (1, 0)), constant_values=b).astype(np.int32)))
    return torch.cat(feats), torch.cat(coords)


def _backbone(name, mode, cuda):
    from detzero_b200 import synthetic
    from detzero_b200.config import AttrDict
    from detzero_b200.det import backbone3d
    cls = getattr(backbone3d, name)
    bb = cls(AttrDict({'NAME': name, 'COMPUTE_MODE': mode}), 5, [1504, 1504, 40]).eval()
    synthetic.load_seeded(bb, 17)
    return bb.to(cuda)


def _collect(monkeypatch, bb, voxels, cuda):
    """(conv module, input tensor, bound arguments, output) of every ops.spconv_fwd call of one eval forward"""
    from detzero_b200.spconv import pytorch as spconv
    calls, ctx = [], []
    orig_fused = spconv._SparseConv.forward_fused

    def fused(self, x, *a, **kw):
        ctx.append((self, x))
        return orig_fused(self, x, *a, **kw)
    orig = ops.spconv_fwd
    sig = inspect.signature(orig)

    def fwd(*args, **kwargs):
        out = orig(*args, **kwargs)
        b = sig.bind(*args, **kwargs)
        b.apply_defaults()
        calls.append((ctx[-1][0], ctx[-1][1], dict(b.arguments), out))
        return out
    monkeypatch.setattr(spconv._SparseConv, 'forward_fused', fused)
    monkeypatch.setattr(ops, 'spconv_fwd', fwd)
    feats, coords = voxels
    with torch.no_grad():
        bb({'voxel_features': feats.to(cuda), 'voxel_coords': coords.to(cuda), 'batch_size': 2})
    torch.cuda.synchronize()
    monkeypatch.undo()
    return calls, orig


def _layer_input(mode, a, cin, n_in):
    """the layer's input as stored, float64 (bf16 modes: its planes summed) and as the (n, P, cin) plane stack"""
    f = a['feats'][:n_in]
    if mode in sa.PLANES:
        P = sa.PLANES[mode]
        planes = f.float().view(n_in, P, -1)[:, :, :cin]
        return planes.to(F64).sum(1), planes
    return f.to(F64), None


#: largest err / bound per (backbone, mode, layer family), printed at the end of the module
RATIOS = {}


def _check_call(mode, conv, x, a, out, variant, fwd=None, rescale=None):
    K, cin, cout = conv.kshape
    n_in = x.num()
    in_sites = x._idx[:n_in]
    nbr, out_sites, _ = pairs_table(in_sites, x.spatial_shape, conv.kernel_size, conv.stride, conv.padding, conv.subm)
    n_out = out_sites.shape[0]
    assert int(a['d_n_out'].item()) == n_out, (conv.indice_key, int(a['d_n_out'].item()), n_out)
    if not conv.subm:
        rule = x.indice_dict[conv.indice_key]
        assert torch.equal(rule.out_idx[:n_out].long(), out_sites), 'strided conv %s: output sites differ' % conv.indice_key
    xr, planes = _layer_input(mode, a, cin, n_in)
    if mode == 'tf32':
        assert torch.equal(xr.float(), sa.rn_tf32(xr.float())), 'a TF32 layer (%s) reads an input that is not TF32-representable' \
            % conv.indice_key
    if rescale is not None:                      # rows rescaled by 10^U(-3, 3), the input re-stored in the layer's format
        s = rescale[:n_in].to(F64)[:, None]
        v = (xr * s).float()
        if mode == 'tf32':
            v = sa.rn_tf32(v)
        feats = a['feats'].clone()
        if mode in sa.PLANES:
            feats[:n_in] = ops.to_planes(v.contiguous(), None, sa.PLANES[mode], _cin_pad(cin))
        else:
            feats[:n_in] = v
        kw = dict(a)
        kw['feats'] = feats
        kw['out'] = None
        out = fwd(**kw)
        a = kw
        xr, planes = _layer_input(mode, a, cin, n_in)
    w = conv.weight.detach().reshape(cout, K, cin).permute(1, 2, 0).to(F64)
    y = sa.conv64(nbr, xr, w)
    A = sa.conv64(nbr, xr.abs(), w.abs())
    sc = a['scale'] if a['scale'] is not None else torch.ones(cout, device=y.device)
    sh = a['shift'] if a['shift'] is not None else torch.zeros(cout, device=y.device)
    o = y * sc.to(F64) + sh.to(F64)
    r_abs = None
    if a['residual'] is not None:
        r = sa.stored_value(mode, a['residual'][:n_out], cout)
        o, r_abs = o + r, r.abs()
    if a['relu']:
        o = o.clamp_min(0)
    got = sa.stored_value(mode, out[:n_out], cout)
    b = sa.bound(mode, K, cin, A, sc, sh, r_abs, got.abs())
    fam = ('subm' if conv.subm else 'strided', K, cin, cout, a['residual'] is not None)
    worst = assert_within(got, o, b, '%s %s %s %s' % (mode, conv.indice_key, fam, variant))
    return fam, worst


@pytest.mark.parametrize('mode', sa.MODES)
@pytest.mark.parametrize('backbone', ['VoxelBackBone8x', 'VoxelResBackBone8x'])
def test_backbone_calls_elementwise(cuda, voxels, monkeypatch, backbone, mode):
    bb = _backbone(backbone, mode, cuda)
    calls, fwd = _collect(monkeypatch, bb, voxels, cuda)
    assert len(calls) >= 10
    g = torch.Generator().manual_seed(5)
    rescale = (10.0 ** (torch.rand(voxels[0].shape[0] * 4, generator=g) * 6 - 3)).to(cuda)
    seen = set()
    for conv, x, a, out in calls:
        for variant, rs in (('as collected', None), ('rows rescaled', rescale)):
            fam, worst = _check_call(mode, conv, x, a, out, variant, fwd=fwd, rescale=rs)
            key = (backbone, mode, fam, variant)
            RATIOS[key] = max(RATIOS.get(key, 0.0), worst)
            seen.add(fam)
    assert any(f[0] == 'strided' and f[1] == 3 for f in seen) and any(f[2] == 5 for f in seen)
    if backbone == 'VoxelResBackBone8x':
        assert any(f[1] == 27 and f[3] == 128 and f[4] for f in seen), 'res4: K = 27, Cout = 128 with a residual'
    del bb
    print('\nlargest err/bound, %s %s:' % (backbone, mode))
    for k in sorted(k for k in RATIOS if k[0] == backbone and k[1] == mode):
        print('  %-40s %-14s %.3g' % (k[2], k[3], RATIOS[k]))


# ---------------------------------------------------------------------------------------------------------------------------------
# c. the TF32 backbone input
# ---------------------------------------------------------------------------------------------------------------------------------
def test_tf32_backbone_input_is_rounded(cuda):
    """conv_input in tf32 on voxel features that are not TF32-representable, with exactly representable weights of one sign: the
    stored output is RNA_tf32(sum RN_tf32(x) w) to the bit.  A truncating read of the raw input gives a smaller sum everywhere"""
    from detzero_b200.spconv import pytorch as spconv
    g = torch.Generator().manual_seed(3)
    shape = [10, 24, 24]
    n = 1500
    flat = torch.randperm(shape[0] * shape[1] * shape[2], generator=g)[:n]
    idx = torch.stack([torch.zeros_like(flat), flat // (shape[1] * shape[2]), (flat // shape[2]) % shape[1], flat % shape[2]], 1).int()
    t = (torch.randint(32, 128, (n, 5), generator=g).float() / 64)             # [0.5, 2), few bits
    ulp = torch.ldexp(torch.ones_like(t), torch.frexp(t).exponent - 11)
    x = t + ulp * (0.55 + 0.3 * torch.rand(n, 5, generator=g))                 # RN rounds up, truncation down
    assert not torch.equal(x, sa.rn_tf32(x))
    conv = spconv.SubMConv3d(5, 16, 3, padding=1, bias=False, indice_key='subm1', mode='tf32')
    with torch.no_grad():
        conv.weight.copy_(torch.randint(1, 5, conv.weight.shape, generator=g).float() / 4)
    conv = conv.to(cuda).eval()
    xt = spconv.SparseConvTensor(x.to(cuda), idx.to(cuda), shape, 1)
    with torch.no_grad():
        y = conv(xt)
    nbr, _, _ = pairs_table(idx.to(cuda), shape, [3, 3, 3], [1, 1, 1], [1, 1, 1], True)
    w = conv.weight.detach().reshape(16, 27, 5).permute(1, 2, 0)
    y64 = sa.conv64(nbr, sa.rn_tf32(x.to(cuda)), w)
    assert torch.equal(y64, y64.float().to(F64))
    want = sa.rna_tf32(y64.float())
    _assert_values(y.features, want, 'conv_input tf32')
    assert y._tf32, "a TF32 layer's output is rounded by its epilogue and passes to the next TF32 layer as it is"


# ---------------------------------------------------------------------------------------------------------------------------------
# d. backward: dgrad (rulebook_transpose + k_spconv_f32), wgrad, SparseInverseConv3d
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def level_tables(cuda, voxels):
    """the real level-1 submanifold table and the level-1 -> level-2 strided table of the two frames, from the rulebook kernels"""
    from detzero_b200.spconv import pytorch as spconv
    feats, coords = voxels
    shape = [41, 1504, 1504]
    x = spconv.SparseConvTensor(feats.to(cuda), coords.to(cuda), shape, 2)
    n1 = x.num()
    nbr1 = ops.rulebook_subm(x._idx, x._count, x._cap, x.grid_index(), [3, 3, 3], layout='k')
    oc, d_n2, _, nbr2, _ = ops.rulebook_conv(x._idx, x._count, x._cap, x.grid_index(), [3, 3, 3], [2, 2, 2], [1, 1, 1],
                                             out_cap=3 * n1, layout='k')
    n2 = int(d_n2.item())
    ref1, _, _ = pairs_table(x._idx[:n1], shape, [3, 3, 3], [1, 1, 1], [1, 1, 1], True)
    ref2, sites2, shape2 = pairs_table(x._idx[:n1], shape, [3, 3, 3], [2, 2, 2], [1, 1, 1], False)
    assert torch.equal(nbr1[:, :n1].long(), ref1) and torch.equal(nbr2[:, :n2].long(), ref2)
    # conv_out's (3, 1, 1) / (2, 1, 1) table on the level-2 sites: K = 3
    ref3, sites3, _ = pairs_table(sites2, shape2, [3, 1, 1], [2, 1, 1], [0, 0, 0], False)
    assert n2 >= 3 * 1024 and sites3.shape[0] >= 3 * 1024
    return dict(n1=n1, n2=n2, sub=(ref1.int().contiguous(), n1, n1), strided=(ref2.int().contiguous(), n2, n1),
                k3=(ref3.int().contiguous(), sites3.shape[0], n2))


def _transpose64(nbr, n_in):
    """nbrT[k][j] = o for every pair (k, j = nbr[k][o], o), -1 elsewhere"""
    K, n_out = nbr.shape
    t = torch.full((K, n_in), -1, dtype=torch.int32, device=nbr.device)
    for k in range(K):
        o = torch.nonzero(nbr[k] >= 0).squeeze(1)
        t[k, nbr[k, o].long()] = o.int()
    return t


def _exact_small(g, shape, dev):
    """values in {0, +-0.25, +-0.5}: products on a 2^-4 grid, every sum of a few thousand of them exact in fp32"""
    v = torch.tensor([0.0, 0.25, -0.25, 0.5, -0.5])
    return v[torch.randint(0, 5, shape, generator=g)].to(dev)


def _fp32_bound(n, A):
    return n * sa.U * (1 + n * sa.U) * A


@pytest.mark.parametrize('exact', [True, False], ids=['exact', 'bounded'])
@pytest.mark.parametrize('table', ['sub', 'strided'])
@pytest.mark.parametrize('cin', [16, 32, 64, 128])
def test_dgrad(cuda, level_tables, table, cin, exact):
    """d_in[j] = sum_k W[k]^T d_out[o] over the pairs: the forward kernel on rulebook_transpose's table, at every width it accepts"""
    nbr, n_out, n_in = level_tables[table]
    K, cout = 27, 32
    g = torch.Generator().manual_seed(cin + (7 if exact else 0))
    if exact:
        dout, w = _exact_small(g, (n_out, cout), cuda), _exact_small(g, (K, cin, cout), cuda)
    else:
        dout = torch.randn(n_out, cout, generator=g).to(cuda) * (10.0 ** (torch.rand(n_out, 1, generator=g) * 6 - 3)).to(cuda)
        w = torch.randn(K, cin, cout, generator=g).to(cuda) / (K * cout) ** 0.5
    d_out = torch.tensor([n_out], dtype=torch.int32, device=cuda)
    d_in = torch.tensor([n_in], dtype=torch.int32, device=cuda)
    nbrT = ops.rulebook_transpose(nbr, d_out, n_in)
    ref_T = _transpose64(nbr, n_in)
    assert torch.equal(nbrT, ref_T)
    got = ops.spconv_fwd(dout, nbrT, d_in, n_in, w.transpose(1, 2).contiguous(), None, None, None, False, _lib.DZ_F32,
                         kshape=(K, cout, cin), layout='k')
    want = sa.conv64(ref_T, dout, w.transpose(1, 2))
    if exact:
        _assert_values(got, want, 'dgrad %s cin=%d' % (table, cin))
    else:
        A = sa.conv64(ref_T, dout.abs(), w.transpose(1, 2).abs())
        assert_within(got, want, _fp32_bound(K * cout + K * 2, A), 'dgrad %s cin=%d' % (table, cin))


@pytest.mark.parametrize('exact', [True, False], ids=['exact', 'bounded'])
@pytest.mark.parametrize('table,cin,cout', [('sub', 5, 16), ('sub', 16, 16), ('strided', 16, 32), ('strided', 64, 64),
                                            ('k3', 128, 128)])
def test_wgrad(cuda, level_tables, table, cin, cout, exact):
    """dW[k] = sum_o in[nbr[k][o]]^T d_out[o]: blocks of 1024 output rows, combined by atomicAdd (>= 3 blocks per offset here);
    cin = 5 (conv_input) and K = 3 (conv_out) included"""
    nbr, n_out, n_in = level_tables[table]
    K = nbr.shape[0]
    assert n_out >= 3 * 1024
    g = torch.Generator().manual_seed(cin * 3 + cout + (1 if exact else 0))
    if exact:
        x, dout = _exact_small(g, (n_in, cin), cuda), _exact_small(g, (n_out, cout), cuda)
    else:
        x = torch.randn(n_in, cin, generator=g).to(cuda)
        dout = torch.randn(n_out, cout, generator=g).to(cuda) * (10.0 ** (torch.rand(n_out, 1, generator=g) * 4 - 2)).to(cuda)
    d_out = torch.tensor([n_out], dtype=torch.int32, device=cuda)
    got = ops.spconv_wgrad(x, nbr, d_out, n_out, dout)
    want = torch.zeros(K, cin, cout, dtype=F64, device=cuda)
    A = torch.zeros_like(want)
    for k in range(K):
        o = torch.nonzero(nbr[k] >= 0).squeeze(1)
        xa, da = x[nbr[k, o].long()].to(F64), dout[o].to(F64)
        want[k] = xa.t() @ da
        A[k] = xa.abs().t() @ da.abs()
    if exact:
        _assert_values(got, want, 'wgrad %s cin=%d cout=%d' % (table, cin, cout))
    else:
        n = n_out + -(-n_out // 1024)        # per element: one FMA per pair, one atomicAdd per block
        assert_within(got, want, _fp32_bound(n, A), 'wgrad %s cin=%d cout=%d' % (table, cin, cout))


def test_inverse_conv_module(cuda, voxels):
    """SparseConv3d (training) then SparseInverseConv3d with its indice_key: output sites = the strided conv's input sites,
    forward and both gradients within the fp32 bound of the pairs restated here"""
    from detzero_b200.spconv import pytorch as spconv
    feats, coords = voxels
    shape = [41, 1504, 1504]
    g = torch.Generator().manual_seed(9)
    down = spconv.SparseConv3d(5, 16, 3, stride=2, padding=1, bias=False, indice_key='sp2').to(cuda).train()
    up = spconv.SparseInverseConv3d(16, 32, 3, indice_key='sp2', bias=False).to(cuda).train()
    x = spconv.SparseConvTensor(feats.to(cuda), coords.to(cuda), shape, 2)
    mid = down(x)
    mid_feat = mid._feat.detach().clone().requires_grad_(True)
    y = up(mid._like(mid_feat))
    n1 = x.num()
    nbr, sites2, _ = pairs_table(x._idx[:n1], shape, [3, 3, 3], [2, 2, 2], [1, 1, 1], False)
    assert torch.equal(y.indices.long(), x._idx[:n1].long())
    T = _transpose64(nbr.int(), n1)
    w = up.weight.detach().reshape(32, 27, 16).permute(1, 2, 0)
    want = sa.conv64(T, mid_feat.detach(), w)
    A = sa.conv64(T, mid_feat.detach().abs(), w.abs())
    assert_within(y.features.detach(), want, _fp32_bound(27 * 16 + 27, A), 'inverse conv forward')
    gy = torch.randn(n1, 32, generator=g).to(cuda)
    y.features.backward(gy)
    want_g = sa.conv64(nbr.int(), gy, w.transpose(1, 2))
    A_g = sa.conv64(nbr.int(), gy.abs(), w.transpose(1, 2).abs())
    assert_within(mid_feat.grad, want_g, _fp32_bound(27 * 32 + 27, A_g), 'inverse conv input gradient')
    dW = torch.zeros(27, 16, 32, dtype=F64, device=cuda)
    AW = torch.zeros_like(dW)
    for k in range(27):
        j = torch.nonzero(T[k] >= 0).squeeze(1)
        a, d = mid_feat.detach()[T[k, j].long()].to(F64), gy[j].to(F64)
        dW[k], AW[k] = a.t() @ d, a.abs().t() @ d.abs()
    got_w = up.weight.grad.reshape(32, 27, 16).permute(1, 2, 0)
    assert_within(got_w, dW, _fp32_bound(n1 + -(-n1 // 1024), AW), 'inverse conv weight gradient')

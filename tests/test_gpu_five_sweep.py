"""The 5-sweep configuration (BASELINE configs[2], ``bench.py --config 3``) at its benchmarked size: ~890 K-point clouds of five
concatenated sweeps, DynamicMeanVFE on the full 1504 x 1504 x 40 lattice -> VoxelResBackBone8x on 6 input channels in the bf16
operand-plane modes -> BEV -> CenterHead, against the CPU oracle chain.

- dynamic voxelization is bit-exact (coordinates, order, count and means) on the full lattice, at every voxel size, and gives the
  same bits on every run;
- a frame with more voxels than the old 400 000 cap comes back whole, through the module and through CenterPoint;
- every (cin_pad, cout) instantiation of the persistent bf16-plane sparse conv, layer by layer with enough tiles that every CTA
  walks at least three of them, against a float64 restatement;
- the whole detector against the oracle, per level and in its detections; eager runs and CUDA-graph replay give the same bits."""
import numpy as np
import pytest
import torch

from oracle import det_ref, spconv_ref
from tests import spconv_arith, util
from tests.test_gpu_bench_config import POST, _check_against_oracle, _settle
from detzero_b200 import _lib

GRID = [1504, 1504, 40]                 # x, y, z
SPARSE_SHAPE = [41, 1504, 1504]         # z, y, x of the backbone's level 1
SMS, TILE_ROWS = 132, 128               # k_spconv_bf16 starts at most one CTA per SM and walks 128-row tiles


def _frame_points(seed, npts=None):
    """bench.run_config3's frame: a batch column in front of the 6 features; padded with far out-of-range points (or cut) to npts"""
    import bench
    p = bench.five_sweep_cloud(seed)
    if npts is not None:
        p = p[:npts] if p.shape[0] >= npts else np.concatenate([p, np.full((npts - p.shape[0], 6), 1.0e4, np.float32)])
    return np.pad(p, ((0, 0), (1, 0))).astype(np.float32)


@pytest.fixture(scope='module')
def frames():
    """the two 5-sweep frames (seeds 0 and 1, the second brought to the first's point count as bench.run_config3 does) and the
    oracle's dynamic voxelization of each"""
    torch.set_num_threads(16)
    p0 = _frame_points(0)
    p1 = _frame_points(1, p0.shape[0])
    out = []
    for p in (p0, p1):
        mean, coords = det_ref.dynamic_mean_vfe(p, util.WAYMO_RANGE, util.VOXEL, GRID)
        out.append(dict(points=p, mean=mean, coords=coords))
    return out


def test_oracle_dynamic_mean_is_a_sequential_float32_sum():
    """pins the target of the bit-exact tests: the oracle's means equal a float32 sum of each voxel's points in point order
    (np.add.at is unbuffered and in order), divided once by the count"""
    torch.set_num_threads(16)
    pts = _frame_points(0)
    mean, coords = det_ref.dynamic_mean_vfe(pts, util.WAYMO_RANGE, util.VOXEL, GRID)
    lo, vs = np.array(util.WAYMO_RANGE[:3], np.float32), np.array(util.VOXEL, np.float32)
    pc = np.floor((pts[:, 1:4] - lo) / vs).astype(np.int64)
    keep = np.all((pc >= 0) & (pc < np.array(GRID)), axis=1)
    pc, data = pc[keep], pts[keep, 1:]
    key = pts[keep, 0].astype(np.int64) * (GRID[0] * GRID[1] * GRID[2]) + (pc[:, 0] * GRID[1] + pc[:, 1]) * GRID[2] + pc[:, 2]
    unq, inv = np.unique(key, return_inverse=True)
    sums = np.zeros((unq.shape[0], data.shape[1]), np.float32)
    np.add.at(sums, inv, data)
    cnt = np.bincount(inv).astype(np.float32)
    assert unq.shape[0] == coords.shape[0] > 300000 and cnt.max() > 20
    assert np.array_equal(mean.numpy().view(np.uint32), (sums / cnt[:, None]).view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------
# a. dynamic voxelization, bit-exact
# ---------------------------------------------------------------------------------------------------------------
def _check_dynamic(cuda, pts, B, want=None):
    """ops.voxelize_dynamic_mean and the DynamicMeanVFE module against the oracle: count, coordinates (in key order) and means
    bit for bit, rows beyond the count zero; a second run gives the same bits"""
    from detzero_b200 import ops
    from detzero_b200.det import cp_modules
    pts = np.ascontiguousarray(pts, np.float32)
    mean_ref, coords_ref = want if want is not None else det_ref.dynamic_mean_vfe(pts, util.WAYMO_RANGE, util.VOXEL, GRID)
    m_ref = coords_ref.shape[0]
    c = pts.shape[1] - 1
    dev_pts = torch.from_numpy(pts).to(cuda)
    runs = []
    for _ in range(2):
        feats, coords, d_m = ops.voxelize_dynamic_mean(dev_pts, c, B, util.WAYMO_RANGE, util.VOXEL, GRID, max(pts.shape[0], 1))
        runs.append((feats.clone(), coords.clone(), d_m.clone()))
    vfe = cp_modules['DynamicMeanVFE'](model_cfg=util.model_cfg('VoxelResBackBone8x').VFE, num_point_features=c, voxel_size=util.VOXEL,
                                       grid_size=GRID, point_cloud_range=util.WAYMO_RANGE)
    bd = vfe({'points': dev_pts, 'batch_size': B})
    runs.append((bd['voxel_features'], bd['voxel_coords'], bd['voxel_count']))
    for feats, coords, d_m in runs:
        m = int(d_m.item())
        assert m == m_ref
        assert feats.shape[0] >= m
        assert torch.equal(coords[:m].cpu(), coords_ref)
        assert np.array_equal(feats[:m].cpu().numpy().view(np.uint32), mean_ref.numpy().view(np.uint32))
        assert torch.all(feats[m:] == 0)
    for feats, coords, d_m in runs[1:]:
        assert torch.equal(feats, runs[0][0]) and torch.equal(coords, runs[0][1])
    return runs[0]


@pytest.mark.gpu
def test_dynamic_voxelization_five_sweep_frame(cuda, frames):
    f = frames[0]
    _check_dynamic(cuda, f['points'], 1, (f['mean'], f['coords']))
    assert f['coords'].shape[0] > 300000


@pytest.mark.gpu
def test_dynamic_voxelization_shuffled_batch_with_an_empty_frame(cuda, frames):
    """three frames whose rows are shuffled together: the key includes b, and a voxel's points are summed in the shuffled order;
    every point of the middle frame is out of range"""
    a = frames[1]['points'].copy()
    mid = frames[0]['points'][::3].copy()
    mid[:, 1] += 200.0
    c = frames[0]['points'].copy()
    a[:, 0], mid[:, 0], c[:, 0] = 0, 1, 2
    pts = np.concatenate([a, mid, c])
    pts = pts[np.random.default_rng(5).permutation(pts.shape[0])]
    feats, coords, d_m = _check_dynamic(cuda, pts, 3)
    b = coords[:int(d_m.item()), 0].cpu()
    assert (b == 0).any() and not (b == 1).any() and (b == 2).any()


@pytest.mark.gpu
def test_dynamic_voxelization_lattice_edges(cuda):
    """duplicates, points exactly on the lattice, x == hi (dropped), points at exactly lo (kept) and one float32 step below lo
    (dropped) on every axis, and an empty input"""
    edge = util.config1_cloud(60000, 3, util.WAYMO_RANGE, c=6)
    lo = np.array(util.WAYMO_RANGE[:3], np.float32)
    g = np.random.default_rng(4)
    at_lo = np.repeat(edge[-12:], 1, axis=0)
    for d in range(3):
        at_lo[2 * d, d] = lo[d]
        at_lo[2 * d + 1, d] = np.nextafter(lo[d], np.float32(-np.inf))
    corner = np.concatenate([lo, g.uniform(0, 1, 3).astype(np.float32)])[None]
    below = corner.copy()
    below[0, :3] = np.nextafter(lo, np.float32(-np.inf))
    pts = np.concatenate([edge, at_lo, corner, corner, below]).astype(np.float32)
    pts = np.pad(pts, ((0, 0), (1, 0)))
    mean_ref, coords_ref = det_ref.dynamic_mean_vfe(pts, util.WAYMO_RANGE, util.VOXEL, GRID)
    assert torch.equal(coords_ref[0], torch.tensor([0, 0, 0, 0], dtype=torch.int32))        # the corner voxel, first in key order
    _check_dynamic(cuda, pts, 1, (mean_ref, coords_ref))
    empty = np.zeros((0, 7), np.float32)
    feats, coords, d_m = _check_dynamic(cuda, empty, 1)
    assert int(d_m.item()) == 0


@pytest.mark.gpu
def test_dynamic_voxelization_one_voxel_of_100k_points(cuda, frames):
    """one voxel holding 100 003 points of features 2^-24 with 1.0 at the middle point: a float32 sum in point order gives other bits
    than one that adds the 1.0 first or reduces pairwise, so only a sequential sum in point order passes"""
    n = 100003
    vox = np.zeros((n, 7), np.float32)
    vox[:, 1:4] = np.array([1.23, -4.56, 0.5], np.float32)
    vox[:, 4:] = np.float32(2.0 ** -24)
    vox[n // 2, 4:] = 1.0
    seq = np.zeros(1, np.float32)
    np.add.at(seq, np.zeros(n, np.int64), vox[:, 4])
    assert np.float32(1.0) + np.float32(2.0 ** -24) == np.float32(1.0)       # adding the 1.0 first leaves exactly 1.0
    assert len({seq[0], np.float32(1.0), np.sum(vox[:, 4], dtype=np.float32)}) == 3
    pts = np.concatenate([frames[0]['points'][:50000], vox])
    mean_ref, coords_ref = det_ref.dynamic_mean_vfe(pts, util.WAYMO_RANGE, util.VOXEL, GRID)
    feats, coords, d_m = _check_dynamic(cuda, pts, 1, (mean_ref, coords_ref))
    lo, vs = np.array(util.WAYMO_RANGE[:3], np.float32), np.array(util.VOXEL, np.float32)
    x, y, z = np.floor((vox[0, 1:4] - lo) / vs).astype(np.int64)
    r = int(np.flatnonzero(np.all(coords_ref.numpy() == np.array([0, z, y, x]), axis=1))[0])
    assert feats[r, 3].item() == np.float32(seq[0] / np.float32(n))


# ---------------------------------------------------------------------------------------------------------------
# b. more voxels than the old 400 000 cap
# ---------------------------------------------------------------------------------------------------------------
def _five_sweep_model(cuda, sp_mode, dense_mode, head_rescale=None):
    import bench
    from detzero_b200 import synthetic
    from detzero_b200.det import build_network
    from detzero_b200.det.dataset import SyntheticWaymoDataset, default_waymo_1sweep_cfg
    dcfg = default_waymo_1sweep_cfg()
    dcfg.POINT_FEATURE_ENCODING.used_feature_list = ['x', 'y', 'z', 'intensity', 'elongation', 'offset']
    ds = SyntheticWaymoDataset(dcfg, synthetic.CLASS_NAMES, training=False, num_frames=1, n_points=bench.N_POINTS)
    model = build_network(bench.make_model_cfg('VoxelResBackBone8x', dense_mode, sp_mode, vfe='DynamicMeanVFE'), 3, ds).eval()
    synthetic.load_seeded(model, 3)
    sd = bench.tune_head_for_bench(model)
    if head_rescale is not None:
        sd = _rescale_head(model, head_rescale)
    return model.to(cuda), sd


def _bd(pts, cuda, i=0):
    return {'points': torch.from_numpy(pts).to(cuda), 'points_per_frame': [pts.shape[0]], 'frame_id': np.array(['s%d' % i]),
            'batch_size': 1}


@pytest.mark.gpu
def test_more_than_400k_voxels_in_one_frame(cuda):
    """600 K points spread uniformly over the lattice: every voxel comes back equal to the oracle, through the module and through
    CenterPoint, which must not report an overflow"""
    g = np.random.default_rng(11)
    lo, hi = np.array(util.WAYMO_RANGE[:3], np.float32), np.array(util.WAYMO_RANGE[3:], np.float32)
    xyz = g.uniform(lo, hi, (600000, 3)).astype(np.float32)
    pts = np.concatenate([np.zeros((600000, 1), np.float32), xyz, g.uniform(0, 1, (600000, 3)).astype(np.float32)], axis=1)
    mean_ref, coords_ref = det_ref.dynamic_mean_vfe(pts, util.WAYMO_RANGE, util.VOXEL, GRID)
    m_ref = coords_ref.shape[0]
    assert m_ref > 550000
    model, _ = _five_sweep_model(cuda, 'bf16', 'tf32')
    _settle(model, lambda: _bd(pts, cuda))           # the first run holds every voxel; the strided levels' hints settle
    with torch.no_grad():
        out = model.forward_device(_bd(pts, cuda))
        model.post_processing(out)                   # no overflow anywhere
    assert int(out['voxel_count'].item()) == m_ref
    assert out['voxel_features'].shape[0] >= m_ref
    assert torch.equal(out['voxel_coords'][:m_ref].cpu(), coords_ref)
    assert np.array_equal(out['voxel_features'][:m_ref].cpu().numpy().view(np.uint32), mean_ref.numpy().view(np.uint32))
    _check_dynamic(cuda, pts, 1, (mean_ref, coords_ref))
    assert int(out['multi_scale_3d_features']['x_conv1']._count.item()) == m_ref


# ---------------------------------------------------------------------------------------------------------------
# c. every bf16-plane instantiation, layer by layer, at production geometry
# ---------------------------------------------------------------------------------------------------------------
#: (name, cin, cout, subm, kernel, stride, padding, residual): the eight (cin_pad, cout) pairs of dz_spconv_fwd_planes as
#: VoxelResBackBone8x runs them on a 5-sweep frame
LAYERS = [('conv_input', 6, 16, True, 3, 1, 1, False), ('res1', 16, 16, True, 3, 1, 1, True), ('res2', 32, 32, True, 3, 1, 1, True),
          ('res3', 64, 64, True, 3, 1, 1, True), ('res4', 128, 128, True, 3, 1, 1, True), ('spconv2', 16, 32, False, 3, 2, 1, False),
          ('spconv3', 32, 64, False, 3, 2, 1, False), ('spconv4', 64, 128, False, 3, 2, (0, 1, 1), False),
          ('conv_out', 128, 128, False, (3, 1, 1), (2, 1, 1), 0, False)]
MIN_ROWS = 3 * SMS * TILE_ROWS          # every CTA of the persistent kernel walks at least three tiles
SPARE = 300                             # capacity rows beyond the count: must be left untouched


def _crop(coords, n):
    """the n sites of the frame's level 1 with the smallest x: a contiguous piece of the real site set"""
    order = np.argsort(coords[:, 3], kind='stable')[:n]
    return coords[np.sort(order)]


@pytest.mark.gpu
@pytest.mark.parametrize('layer', LAYERS, ids=[l[0] for l in LAYERS])
def test_plane_kernel_layer_at_scale(cuda, frames, layer):
    """module path (forward_fused, scheduled; tile-major table in the bf16 modes) in every compute mode against a float64
    restatement on the same input, element by element within the bounds of tests/spconv_arith.py; in the bf16 modes scheduled,
    unscheduled and tile-major launches give the same bits and capacity rows beyond the count are untouched"""
    from detzero_b200 import ops
    from detzero_b200.spconv import pytorch as spconv
    name, cin, cout, subm, ks, stride, pad, res = layer
    coords = frames[0]['coords'].numpy()
    n_in = min(coords.shape[0], 60000 if subm else 120000)
    while True:
        idx = _crop(coords, n_in)
        if subm:
            pairs, n_out, out_idx = spconv_ref.rulebook_subm(idx, SPARSE_SHAPE, ks), n_in, idx
        else:
            out_idx, _, pairs = spconv_ref.rulebook_conv(idx, SPARSE_SHAPE, ks, stride, pad)
            n_out = out_idx.shape[0]
        if n_out >= MIN_ROWS + TILE_ROWS or n_in == coords.shape[0]:
            break
        n_in = min(coords.shape[0], n_in * 2)
    assert -(-n_out // TILE_ROWS) >= 3 * SMS, (name, n_out)
    g = np.random.default_rng(cin * 1000 + cout + (0 if subm else 7))
    f = torch.from_numpy(g.normal(0, 1, (n_in, cin)).astype(np.float32))
    kshape = [ks] * 3 if isinstance(ks, int) else list(ks)
    w = torch.from_numpy(g.normal(0, 1.0 / np.sqrt(np.prod(kshape) * cin), (cout, *kshape, cin)).astype(np.float32))
    scale = torch.from_numpy(g.uniform(0.5, 1.5, cout).astype(np.float32))
    shift = torch.from_numpy(g.normal(0, 0.1, cout).astype(np.float32))
    r = torch.from_numpy(g.normal(0, 1, (n_out, cout)).astype(np.float32)) if res else None
    K = int(np.prod(kshape))
    native = {}

    def reference(mode):
        """float64 x . w epilogue of the layer's input and residual as the mode stores them (bf16: the planes, summed; tf32: the
        input RN-rounded once) and sum |x| |w|"""
        kind = mode if mode in ('bf16x2', 'bf16', 'tf32') else 'fp32'
        if kind not in native:
            if kind in spconv_arith.PLANES:
                fs = torch.stack(spconv_arith.split_bf16(f)[:spconv_arith.PLANES[kind]]).double().sum(0)
            else:
                fs = (spconv_arith.rn_tf32(f) if kind == 'tf32' else f).double()
            native[kind] = (spconv_ref.sparse_conv_native(fs, w.double(), pairs, n_out),
                            spconv_ref.sparse_conv_native(fs.abs(), w.double().abs(), pairs, n_out))
        y, A = native[kind]
        rs = None
        if res:
            rs = sum(p.double() for p in spconv_arith.residual_pieces(mode, r))
        want = y * scale.double() + shift.double() + (0 if rs is None else rs)
        return torch.relu(want), A, (None if rs is None else rs.abs())
    cap = n_in + (SPARE if subm else 0)
    fc = torch.full((cap, cin), 1e3)
    fc[:n_in] = f
    ic = torch.zeros((cap, 4), dtype=torch.int32)
    ic[:n_in] = torch.from_numpy(idx)
    d_n = torch.tensor([n_in], dtype=torch.int32, device=cuda)
    for mode in spconv_arith.MODES:
        if mode not in _lib.MODES:
            pytest.skip('mode %s not built' % mode)
        P = _lib.PLANES.get(_lib.MODES[mode], 0)
        x = spconv.SparseConvTensor(fc.to(cuda), ic.to(cuda), SPARSE_SHAPE, 1, count=d_n, n_host=n_in)
        if subm:
            conv = spconv.SubMConv3d(cin, cout, ks, bias=False, indice_key='k', mode=mode)
        else:
            conv = spconv.SparseConv3d(cin, cout, ks, stride=stride, padding=pad, bias=False, indice_key='k', mode=mode)
        with torch.no_grad():
            conv.weight.copy_(w)
        conv = conv.to(cuda)
        resid = None
        if res:
            rc = torch.full((cap, cout), -1e3)
            rc[:n_out] = r
            resid = x._like(rc.to(cuda))
        sc, sh = scale.to(cuda), shift.to(cuda)
        with torch.no_grad():
            y = conv.forward_fused(x, sc, sh, resid, True)
        rule = x.indice_dict['k']
        if mode != 'fp32':                                                       # the module ran the scheduled (tile-major) path
            assert rule.order is not None and (rule.tab_tiles is not None or not P), name
        d_out = x._count if subm else rule.d_n_out
        out_cap = x._cap if subm else rule.out_cap
        assert int(d_out.item()) == n_out
        if not subm:
            assert np.array_equal(rule.out_idx[:n_out].cpu().numpy(), out_idx), name
        got = y.features.cpu()
        assert got.shape == (n_out, cout)
        want, A, r_abs = reference(mode)
        util.assert_within(got, want, spconv_arith.bound(mode, K, cin, A, scale, shift, r_abs, got.double().abs()),
                           '%s %s' % (name, mode))
        if not P:
            continue
        # the same launch unscheduled, scheduled, and scheduled from the tile-major table: bit for bit, spare rows untouched
        fp = x._as_planes(P, 8 if cin <= 8 else cin)
        rp = None if resid is None else resid._as_planes(P, cout)
        wp = conv.packed_weight(_lib.MODES[mode])
        outs = []
        for kw in ({}, {'row_order': rule.order}, {'row_order': rule.order, 'tab_tiles': rule.tab_tiles}):
            o = torch.full((out_cap + SPARE, P * cout), -7.0, device=cuda, dtype=torch.bfloat16)
            ops.spconv_fwd(fp, rule.tab, d_out, out_cap, wp, sc, sh, rp, True, _lib.MODES[mode], kshape=conv.kshape, layout='row',
                           out=o[:out_cap], d_n_in=None if subm else x._count, **kw)
            outs.append(o)
            assert torch.all(o[n_out:] == -7.0), (name, mode, kw.keys())
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), (name, mode)
        assert torch.equal(outs[2][:n_out], y._feat[:n_out]), (name, mode)


# ---------------------------------------------------------------------------------------------------------------
# d. the whole detector at config 3 against the oracle
# ---------------------------------------------------------------------------------------------------------------
HEAD = 'dense_head.heads_list.0.%s.1.'
HEADS = ['center', 'center_z', 'dim', 'rot', 'iou', 'hm']
#: per head: the (low, high) values the central 98 % of each output channel is mapped to -- cell offsets within a cell, heights
#: and log sizes of objects a few metres across, unit sin / cos and IoU logits
HEAD_RANGE = {'center': (-0.5, 0.5), 'center_z': (-1.0, 2.0), 'dim': (-0.5, 1.5), 'rot': (-1.0, 1.0), 'iou': (-1.0, 1.0)}
PER_CLASS = 500                          # heatmap cells per class above SCORE_THRESH after the rescale


def _rescale_head(model, rescale):
    """every CenterHead output o' = alpha * (o - b) + beta per channel: the last (linear) conv of each head with its weights scaled
    by alpha and its bias set to beta"""
    sd = model.state_dict()
    with torch.no_grad():
        for n, (alpha, beta) in rescale.items():
            sd[HEAD % n + 'weight'].mul_(alpha.view(-1, 1, 1, 1).to(sd[HEAD % n + 'weight']))
            sd[HEAD % n + 'bias'].copy_(beta)
    return {k: v.detach().clone() for k, v in model.state_dict().items()}


def _head_rescale_for(maps, sd):
    """bench.tune_head_for_bench calibrates the seeded head on 1-sweep frames.  On a 5-sweep frame its outputs run far out of
    range: every box the oracle keeps scores exactly 1.0, ~27 K cells pass SCORE_THRESH against the 4096 of NMS_PRE_MAXSIZE, log
    sizes reach -46 .. 7 (boxes of 1e-14 .. 1000 m) and centre offsets +-50 cells.  Which boxes come out is then decided by exact
    score ties and by NMS cascades among kilometre-sized boxes, not by the network's features.  Map every output channel
    affinely into the range a trained head produces (HEAD_RANGE), and the heatmap so that each class's PER_CLASS-th largest logit
    sits at SCORE_THRESH and its largest at sigmoid = 0.95 (~1.5 K candidates, as bench.tune_head_for_bench aims for)."""
    out = {}
    for n in HEADS:
        z = maps[n][0].double().flatten(1) - sd[HEAD % n + 'bias'].double()[:, None]        # (channels, cells): W * h
        if n == 'hm':
            top = z.topk(PER_CLASS, dim=1)[0]
            lo_t, hi_t = float(np.log(POST['SCORE_THRESH'] / (1 - POST['SCORE_THRESH']))), float(np.log(0.95 / 0.05))
            lo, hi = top[:, -1], top[:, 0]
        else:
            lo_t, hi_t = HEAD_RANGE[n]
            lo, hi = torch.quantile(z, 0.01, dim=1), torch.quantile(z, 0.99, dim=1)
        alpha = (hi_t - lo_t) / (hi - lo)
        out[n] = (alpha.float(), (lo_t - alpha * lo).float())
    return out


def _oracle_chain(sd, f, heads_only_from=None):
    with torch.no_grad():
        if heads_only_from is None:
            lv = det_ref.voxel_backbone(sd, 'backbone3d.', f['mean'], f['coords'].numpy(), SPARSE_SHAPE, 1, res=True)
            s2d = det_ref.bev_backbone(sd, 'backbone2d.', det_ref.height_compression(lv['out']), [5, 5], [1, 2], [1, 2])
        else:
            lv, s2d = heads_only_from
        maps = det_ref.center_head_maps(sd, 'dense_head.', s2d, HEADS)
        boxes = det_ref.generate_predicted_boxes(maps, util.WAYMO_RANGE, util.VOXEL, 8, POST, use_iou=True)[0]
    return lv, s2d, maps, boxes


@pytest.fixture(scope='module')
def world(cuda, frames):
    """the oracle chain of both frames: dynamic mean VFE -> VoxelResBackBone8x (6 input channels) -> height compression -> BEV ->
    CenterHead -> decode + NMS, with the bench weights and the head outputs rescaled for 5-sweep frames (_head_rescale_for)"""
    _, sd = _five_sweep_model(cuda, 'bf16', 'tf32')
    torch.set_num_threads(16)
    lv0, s2d0, maps0, boxes0 = _oracle_chain(sd, frames[0])
    assert float(boxes0['pred_scores'].min()) == 1.0                  # the bench calibration saturates on this frame
    rescale = _head_rescale_for(maps0, sd)
    _, sd = _five_sweep_model(cuda, 'bf16', 'tf32', rescale)
    out = []
    for i, f in enumerate(frames):
        pre = (lv0, s2d0) if i == 0 else None
        lv, s2d, maps, boxes = _oracle_chain(sd, f) if pre is None else _oracle_chain(sd, f, pre)
        assert 100 < boxes['pred_boxes'].shape[0] < POST['NMS_POST_MAXSIZE'], i
        assert float(boxes['pred_scores'].max()) < 0.99, i
        out.append(dict(levels=lv, boxes=boxes))
    return dict(frames=out, rescale=rescale)


@pytest.mark.gpu
@pytest.mark.parametrize('sp_mode,dense_mode', [('bf16x2', 'fp32'), ('bf16', 'tf32')])
def test_five_sweep_detector_vs_oracle(cuda, frames, world, sp_mode, dense_mode):
    """per level within LEVEL_TOL; detections: >= 90 % of the boxes within 5 cm / 0.05 rad / 0.02 score, for bf16x2 sparse + fp32
    dense and for bf16 sparse + TF32 dense (the benchmarked pair).  The score bounds of DET_TOL are not used here: the seeded head
    is steep on these frames, and turns feature differences of 9e-7 (fp32) and 6e-5 (bf16x2) relative to the oracle's into score
    differences of 1.5e-5 and 3e-4 (H100), above DET_TOL's 1e-5 and 1e-4."""
    if sp_mode not in _lib.MODES:
        pytest.skip('mode %s not built' % sp_mode)
    model, _ = _five_sweep_model(cuda, sp_mode, dense_mode, world['rescale'])
    for i, f in enumerate(frames):
        _settle(model, lambda: _bd(f['points'], cuda, i))
        with torch.no_grad():
            bd = model.forward_device(_bd(f['points'], cuda, i))
            pred, _ = model.post_processing(bd)
        _check_against_oracle({'frames': {i: world['frames'][i]}}, sp_mode, bd, pred, [i], dense_exact=False)


# ---------------------------------------------------------------------------------------------------------------
# e. replay of the whole detector at config 3
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_five_sweep_graph_replay_is_bit_exact(cuda, frames):
    """eager twice, then CUDA-graph replay over both frames twice: final boxes and the `out` features are the same bits every time"""
    model, _ = _five_sweep_model(cuda, 'bf16', 'tf32')
    for i, f in enumerate(frames):
        _settle(model, lambda: _bd(f['points'], cuda, i))
    eager = []
    with torch.no_grad():
        for rep in range(2):
            for i, f in enumerate(frames):
                o = model.forward_device(_bd(f['points'], cuda, i))
                model.post_processing(o)
                t = o['encoded_spconv_tensor']
                n = int(t._count.item())
                got = (o['final_boxes_padded'].clone(), o['final_boxes_count'].clone(), t._feat[:n].clone())
                if rep == 0:
                    eager.append(got)
                else:
                    assert all(torch.equal(a, b) for a, b in zip(got, eager[i])), i
    assert int(eager[0][1].sum().item()) > 0
    static = _bd(frames[0]['points'], cuda)
    g, out = model.capture_graph(static, warmup=1)
    for rep in range(2):
        for i, f in enumerate(frames):
            static['points'].copy_(torch.from_numpy(f['points']))
            g.replay()
            model.post_processing(out)
            t = out['encoded_spconv_tensor']
            n = int(t._count.item())
            assert torch.equal(out['final_boxes_count'], eager[i][1]), (rep, i)
            assert torch.equal(out['final_boxes_padded'], eager[i][0]), (rep, i)
            assert n == eager[i][2].shape[0] and torch.equal(t._feat[:n], eager[i][2]), (rep, i)

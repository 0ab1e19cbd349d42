"""Refiner inputs built on the device (detzero_b200/refine/data.py, csrc/refine_data.cu) against the float64 oracle
(oracle/refine_data_ref.py) on a synthetic sequence at Waymo-like world offsets (~5 km): crop counts, keyed selections, features,
revert, determinism, batch independence, the per-object-pickle path and the refiner forward on the built inputs."""
import numpy as np
import pytest
import torch

from detzero_b200 import synthetic
from detzero_b200.refine import data as D
from oracle import refine_data_ref as R
from oracle import weights

pytestmark = pytest.mark.gpu
SEED = 21
COORD_TOL = 5e-5          # metres, columns derived from coordinates (xyz, p2co, p2s)


def _seq(tracks=10, frames=24, lengths=None, n_background=20000, seed=3):
    return synthetic.synthetic_sequence(seed, frames=frames, tracks=tracks, n_background=n_background, lengths=lengths)


def _dev(s, cuda):
    tb = D.TrackBatch(s['boxes'], s['frame_of_box'], s['scores'], s['box_num'], s['cls'], s['track_uid'], cuda)
    return torch.from_numpy(s['frames']).to(cuda), s['frame_offsets'], torch.from_numpy(s['poses']).to(cuda), tb


BUILD = {'prm': D.position_inputs, 'crm': D.confidence_inputs, 'grm': D.geometry_inputs}


def _cmp_p2co(got, want, C, where):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    coord = list(range(3)) + list(range(4, 31))
    err = np.abs(got[..., coord] - want[..., coord]).max() if got.size else 0.0
    assert err <= COORD_TOL, (where, err)
    exact = [3] + list(range(31, C))
    assert np.array_equal(got[..., exact], np.asarray(want[..., exact], np.float32)), where


@pytest.fixture(scope='module')
def seq():
    return _seq(lengths=[24, 1, 2, 17, 24, 5, 9, 24, 3, 12])


@pytest.mark.parametrize('kind', ['prm', 'crm', 'grm'])
def test_inputs_match_oracle(cuda, seq, kind):
    s = seq
    frames, off, poses, tb = _dev(s, cuda)
    cfg = None
    with_class = False
    if kind == 'prm':
        cfg = dict(D.prm_data_cfg(), ENCODING=D.P2CO_CLASS)
        with_class = True
    out = BUILD[kind](frames, off, poses, tb, cfg=cfg, seed=SEED, return_selection=True)
    ref = R.build_batch(kind, s['frames'], s['frame_offsets'], s['poses'], s, SEED, with_class=with_class)
    counts, sel = out['crop_counts'].cpu().numpy(), out['selection'].cpu().numpy()
    for b, r in enumerate(ref):
        L = int(s['box_num'][b])
        assert np.array_equal(counts[b, :L], r['counts']), b
        if kind == 'prm':
            C = 35
            got = sel[b].reshape(200, 256 + 48)
            for j in range(L):
                assert np.array_equal(got[j, :len(r['sel'][0][j])], r['sel'][0][j])
                assert np.array_equal(got[j, 256:256 + len(r['sel'][1][j])], r['sel'][1][j])
            _cmp_p2co(out['pos_query_points'][b].cpu(), r['pos_query_points'], C, ('q', b))
            _cmp_p2co(out['pos_memory_points'][b].cpu(), r['pos_memory_points'], C, ('m', b))
            assert np.all(out['pos_query_points'][b, L:].cpu().numpy() == 0)
            assert np.abs(out['pos_trajectory'][b].cpu().numpy() - r['pos_trajectory']).max() <= COORD_TOL
            assert np.array_equal(out['padding_mask'][b].cpu().numpy(), r['padding_mask'].astype(np.float32))
            assert np.abs(out['pos_init_box'][b].cpu().numpy()[[3, 4, 5, 6]] - r['pos_init_box'][[3, 4, 5, 6]]).max() <= 1e-6
        elif kind == 'crm':
            got = sel[b].reshape(200, 256)
            for j in range(L):
                assert np.array_equal(got[j, :len(r['sel'][j])], r['sel'][j])
            _cmp_p2co(out['conf_points'][b].cpu(), r['conf_points'], 32, ('c', b))
            assert np.array_equal(out['conf_score'][b].cpu().numpy(), r['conf_score'].astype(np.float32))
        else:
            nq = r['geo_query_num']
            assert int(out['geo_query_num'][b]) == nq
            for i in range(nq):
                assert np.array_equal(sel[b, i * 256:i * 256 + len(r['sel'][0][i])], r['sel'][0][i])
            assert np.array_equal(sel[b, 768:768 + len(r['sel'][1])], r['sel'][1])
            q = out['geo_query_points'][b].cpu().numpy()
            assert np.abs(q[:nq, :, :3] - r['geo_query_points'][:, :, :3]).max() <= COORD_TOL
            assert np.array_equal(q[:nq, :, 3], r['geo_query_points'][:, :, 3].astype(np.float32))
            assert np.all(q[nq:] == 0)
            assert np.array_equal(out['geo_query_boxes'][b, :nq].cpu().numpy(), r['geo_query_boxes'].astype(np.float32))
            m = out['geo_memory_points'][b].cpu().numpy()
            coord = [0, 1, 2, 4, 5, 6, 7, 8, 9]
            assert np.abs(m[:, coord] - r['geo_memory_points'][:, coord]).max() <= COORD_TOL
            assert np.array_equal(m[:, [3, 10]], r['geo_memory_points'][:, [3, 10]].astype(np.float32))


def test_revert_matches_oracle(cuda, seq):
    s = seq
    _, _, poses, tb = _dev(s, cuda)
    g = np.random.default_rng(1)
    pred = np.concatenate([g.normal(0, 5, (10, 200, 3)), g.uniform(0.5, 5, (10, 200, 3)), g.uniform(-4, 4, (10, 200, 1))], 2)
    pred = pred.astype(np.float32)
    lid, wor = D.revert_position_boxes(torch.from_numpy(pred).to(cuda), poses, tb)
    gpred = pred[:, 0, :]
    glid, gwor = D.revert_geometry_boxes(torch.from_numpy(gpred).to(cuda), poses, tb)
    for b in range(10):
        L = int(s['box_num'][b])
        bp = s['poses'][s['frame_of_box'][b, :L]]
        for (dl, dw), (rl, rw) in (((lid, wor), R.revert_position(pred[b], s['boxes'][b], L, bp)),
                                   ((glid, gwor), R.revert_geometry(gpred[b], s['boxes'][b], L, bp))):
            for got, want in ((dl[b, :L].cpu().numpy(), rl), (dw[b, :L].cpu().numpy(), rw)):
                assert np.abs(got[:, :6] - want[:, :6]).max() <= 1e-4
                assert np.abs(got[:, 6] - want[:, 6]).max() <= 1e-5
            assert np.all(dl[b, L:].cpu().numpy() == 0)


def test_deterministic_and_batch_independent(cuda):
    s = _seq(tracks=64, frames=16, n_background=8000, seed=5)
    frames, off, poses, tb = _dev(s, cuda)
    for kind, fn in BUILD.items():
        a = fn(frames, off, poses, tb, seed=SEED)
        b2 = fn(frames, off, poses, tb, seed=SEED)
        for k in a:
            assert torch.equal(a[k], b2[k]), (kind, k)
        for b in range(64):
            one = fn(frames, off, poses, tb.select([b]), seed=SEED)
            for k in one:
                if kind == 'grm' and k in ('geo_query_points', 'geo_query_boxes'):
                    n = one[k].shape[1]
                    assert torch.equal(one[k][0], a[k][b, :n]) and not a[k][b, n:].any(), (kind, k, b)
                else:
                    assert torch.equal(one[k][0], a[k][b]), (kind, k, b)


def test_object_infos_path(cuda, seq):
    s = seq
    infos = []
    for b in range(10):
        L = int(s['box_num'][b])
        crops = R.track_crops(s['frames'], s['frame_offsets'], s['poses'], s['boxes'][b], s['frame_of_box'][b], L)
        infos.append({'obj_id': str(b), 'name': ['Vehicle', 'Pedestrian', 'Cyclist'][int(s['cls'][b]) - 1],
                      'boxes_global': s['boxes'][b, :L], 'score': s['scores'][b, :L], 'pose': s['poses'][s['frame_of_box'][b, :L]],
                      'pts': [np.concatenate([c[:, :3] + s['boxes'][b, j, :3], c[:, 3:4]], 1) for j, c in enumerate(crops)]})
    ff, foff, fposes, ftb = D.tracks_from_object_infos(infos, track_uid=s['track_uid'], device=cuda)
    frames, off, poses, tb = _dev(s, cuda)
    for kind, fn in BUILD.items():
        a = fn(frames, off, poses, tb, seed=SEED, return_selection=True)
        o = fn(ff, foff, fposes, ftb, seed=SEED, crop=False, return_selection=True)
        assert torch.equal(a['crop_counts'], o['crop_counts']) and torch.equal(a['selection'], o['selection']), kind
        for k in a:
            if a[k].dtype == torch.float32:
                assert (a[k] - o[k]).abs().max().item() <= 1e-5, (kind, k)


def test_forward_on_device_inputs(cuda, seq):
    """the refiner modules (fp32 kernels) on device-built inputs vs on the uploaded oracle inputs"""
    from detzero_b200.refine import ConfidencePointnet, GeometryTransformer, PositionTransformer
    s = seq
    frames, off, poses, tb = _dev(s, cuda)
    up = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.float32, device=cuda)
    report = {}
    cfg = synthetic.prm_cfg(); cfg.COMPUTE_MODE = 'fp32'
    m = PositionTransformer(cfg, 32, 32).eval(); weights.load_seeded(m, SEED); m = m.to(cuda)
    dev = D.position_inputs(frames, off, poses, tb, seed=SEED)
    ref = R.build_batch('prm', s['frames'], s['frame_offsets'], s['poses'], s, SEED)
    o = {k: up(np.stack([r[k] for r in ref])) for k in ('pos_query_points', 'pos_memory_points', 'pos_trajectory', 'padding_mask')}
    a, b = m(dict(dev))['batch_box_preds'], m(o)['batch_box_preds']
    valid = dev['padding_mask'] == 0
    report['prm'] = (a[valid][:, :6] - b[valid][:, :6]).abs().max().item()
    assert report['prm'] <= 1e-3
    cfg = synthetic.grm_cfg(); cfg.COMPUTE_MODE = 'fp32'
    m = GeometryTransformer(cfg, 11, 4).eval(); weights.load_seeded(m, SEED + 1); m = m.to(cuda)
    dev = D.geometry_inputs(frames, off, poses, tb, seed=SEED)
    ref = R.build_batch('grm', s['frames'], s['frame_offsets'], s['poses'], s, SEED)
    Q = dev['geo_query_points'].shape[1]
    qp = np.zeros((10, Q, 256, 4)); qb = np.zeros((10, Q, 7))
    for i, r in enumerate(ref):
        qp[i, :r['geo_query_num']], qb[i, :r['geo_query_num']] = r['geo_query_points'], r['geo_query_boxes']
    o = {'geo_query_points': up(qp), 'geo_query_boxes': up(qb), 'geo_memory_points': up(np.stack([r['geo_memory_points'] for r in ref])),
         'geo_query_num': torch.tensor([r['geo_query_num'] for r in ref], device=cuda)}
    a, b = m(dict(dev))['batch_box_preds'], m(o)['batch_box_preds']
    report['grm'] = (a - b).abs().max().item()
    assert report['grm'] <= 1e-3
    cfg = synthetic.crm_cfg(); cfg.COMPUTE_MODE = 'fp32'
    m = ConfidencePointnet(cfg, 32, 32).eval(); weights.load_seeded(m, SEED + 2); m = m.to(cuda)
    dev = D.confidence_inputs(frames, off, poses, tb, seed=SEED)
    ref = R.build_batch('crm', s['frames'], s['frame_offsets'], s['poses'], s, SEED)
    a = m(dict(dev))['pred_score']
    b = m({'conf_points': up(np.stack([r['conf_points'] for r in ref])), 'conf_score': up(np.stack([r['conf_score'] for r in ref])),
           'box_num': dev['box_num']})['pred_score']
    report['crm'] = (a - b).abs().max().item()
    assert report['crm'] <= 1e-4
    print('forward on device vs oracle inputs, max |diff|:', report)


def test_edge_cases(cuda):
    """a frame with zero points, a track whose crops are all empty, B = 1"""
    s = _seq(tracks=3, frames=6, lengths=[6, 3, 1], n_background=3000, seed=9)
    F = len(s['poses'])
    s['frame_offsets'] = np.append(s['frame_offsets'], s['frame_offsets'][-1])          # frame F: no points
    s['poses'] = np.concatenate([s['poses'], s['poses'][:1]], 0)
    s['frame_of_box'][2, 0] = F
    s['boxes'][1, :3, 0] += 2000.0                                                       # far from every point
    frames, off, poses, tb = _dev(s, cuda)
    for kind, fn in BUILD.items():
        out = fn(frames, off, poses, tb, seed=SEED, return_selection=True)
        ref = R.build_batch(kind, s['frames'], s['frame_offsets'], s['poses'], s, SEED)
        assert ref[1]['counts'].sum() == 0 and ref[2]['counts'].sum() == 0
        for b in range(3):
            assert np.array_equal(out['crop_counts'][b, :int(s['box_num'][b])].cpu().numpy(), ref[b]['counts'])
        one = fn(frames, off, poses, tb.select([1]), seed=SEED)
        for k in one:
            if kind == 'grm' and k in ('geo_query_points', 'geo_query_boxes'):
                continue
            assert torch.equal(one[k][0], out[k][1]), (kind, k)
    out = D.position_inputs(frames, off, poses, tb.select([2]), seed=SEED)
    ref = R.build_batch('prm', s['frames'], s['frame_offsets'], s['poses'], {k: (v[2:3] if isinstance(v, np.ndarray) and v.ndim and
                                                                                len(v) == 3 else v) for k, v in s.items()}, SEED)
    _cmp_p2co(out['pos_query_points'][0].cpu(), ref[0]['pos_query_points'], 32, 'single')

"""Refiner training samples built on the device (refine.data.crop_tracks, geometry_training_inputs, confidence_training_inputs,
training_order; csrc/refine_data.cu) against the float64 oracle (oracle/refine_train_data_ref.py) on synthetic sequences at Waymo-like
world offsets (~5 km): the keyed draws exactly, the features within test_gpu_refine_data.py's tolerances, the crop-once path bit
for bit, batch-order / chunk / repeat independence, the rejections, the workspaces of the new entry points, and one training step
of each model on samples built from a tracked, assigned and refined sequence."""
import numpy as np
import pytest
import torch

from detzero_b200 import _lib, ops, synthetic
from detzero_b200.config import AttrDict
from detzero_b200.refine import data as D
from detzero_b200.refine import score as S
from detzero_b200.refine.modules import RefineTemplate
from detzero_b200.track import assign_track_target, ground_truth_from_infos, track_sequences
from oracle import refine_data_ref as R
from oracle import refine_train_data_ref as T
from oracle import refine_inputs as ri
from oracle import weights
from tests.test_gpu_workspace import _blank, check_workspace

pytestmark = pytest.mark.gpu
SEED, EPOCH = 21, 4
COORD_TOL = 5e-5          # metres, columns derived from coordinates (xyz, p2co, p2s)
LOSS_TOL = 5e-3           # tf32 step losses, relative (tests/test_gpu_grm_train.py, test_gpu_refine_train.py)
L_ = _lib.lib
P = ops._p


def _targets(s, cuda, seed=2):
    """TrackTargets of a synthetic sequence: ground truth near each box, some unmatched slots, every track a matched tracklet with a
    matched box; and (B, L) IoU labels with -1 padding"""
    g = np.random.default_rng(seed)
    B, L = s['boxes'].shape[:2]
    valid = np.arange(L)[None, :] < np.asarray(s['box_num'])[:, None]
    matched = valid & (g.random((B, L)) < 0.8)
    matched[:, 0] |= valid[:, 0]
    gt = s['boxes'] + np.concatenate([g.normal(0, 0.1, (B, L, 3)), g.normal(0, 0.05, (B, L, 3)), g.normal(0, 0.02, (B, L, 1))], 2)
    gt[~matched] = 0
    t = lambda a, dt: torch.as_tensor(a, dtype=dt, device=cuda)  # noqa: E731
    tg = D.TrackTargets(t(gt, torch.float64), t(matched, torch.uint8), t(np.ones(B), torch.uint8), t(np.ones(B), torch.int32),
                        t(np.zeros((B, L, 7)), torch.float32), t(np.arange(B), torch.int32))
    iou = np.where(valid, g.uniform(0, 1, (B, L)), -1).astype(np.float32)
    return tg, t(iou, torch.float32)


def _dev(s, cuda):
    tb = D.TrackBatch(s['boxes'], s['frame_of_box'], s['scores'], s['box_num'], s['cls'], s['track_uid'], cuda)
    return torch.from_numpy(s['frames']).to(cuda), s['frame_offsets'], torch.from_numpy(s['poses']).to(cuda), tb


@pytest.fixture(scope='module')
def seq():
    s = synthetic.synthetic_sequence(3, frames=24, tracks=10, n_background=20000, lengths=[24, 1, 2, 17, 24, 5, 9, 24, 3, 12])
    tg, iou = _targets(s, 'cuda')
    return s, tg, iou


def _build(kind, frames, off, poses, tb, tg, iou, crop=True, epoch=EPOCH, **kw):
    if kind == 'grm':
        return D.geometry_training_inputs(frames, off, poses, tb, tg, seed=SEED, epoch=epoch, crop=crop, return_selection=True, **kw)
    return D.confidence_training_inputs(frames, off, poses, tb, iou, seed=SEED, epoch=epoch, crop=crop, return_selection=True, **kw)


def _cmp(got, want, coord, exact, where):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    err = np.abs(got[..., coord] - want[..., coord]).max() if got.size else 0.0
    assert err <= COORD_TOL, (where, err)
    assert np.array_equal(got[..., exact], np.asarray(want[..., exact], np.float32)), where


def check_against_oracle(kind, out, s, tg, iou):
    ref = T.build_train_batch(kind, s['frames'], s['frame_offsets'], s['poses'], s, SEED, EPOCH, gt_boxes=tg.gt_boxes.cpu().numpy(),
                              matched=tg.matched.cpu().numpy(), iou=iou.cpu().numpy())
    kept, counts, sel = out['kept'].cpu().numpy(), out['crop_counts'].cpu().numpy(), out['selection'].cpu().numpy()
    for b, r in enumerate(ref):
        n = len(r['kept'])
        assert np.array_equal(kept[b, :n], r['kept']) and (kept[b, n:] == -1).all(), b
        assert np.array_equal(counts[b, :n], r['counts']), b
        if kind == 'grm':
            nq = r['geo_query_num']
            assert int(out['kept_num'][b]) == n and int(out['geo_query_num'][b]) == nq
            qs = out['query_slots'][b].cpu().numpy()
            assert np.array_equal(qs[:nq], r['query_slots']) and (qs[nq:] == -1).all()
            assert np.array_equal(out['flip'][b, :n].cpu().numpy(), r['flip']) and not out['flip'][b, n:].any()
            for i in range(nq):
                assert np.array_equal(sel[b, i * 256:i * 256 + len(r['sel'][0][i])], r['sel'][0][i])
            assert np.array_equal(sel[b, 768:768 + len(r['sel'][1])], r['sel'][1])
            q = out['geo_query_points'][b].cpu().numpy()
            _cmp(q[:nq], r['geo_query_points'], [0, 1, 2], [3], ('q', b))
            assert not q[nq:].any()
            for k in ('geo_query_boxes', 'gt_geo_query_boxes'):
                v = out[k][b].cpu().numpy()
                assert np.array_equal(v[:nq], r[k].astype(np.float32)) and not v[nq:].any(), (k, b)
            _cmp(out['geo_memory_points'][b].cpu(), r['geo_memory_points'], [0, 1, 2, 4, 5, 6, 7, 8, 9], [3, 10], ('m', b))
            for k in ('geo_trajectory', 'gt_geo_trajectory'):
                v = out[k][b].cpu().numpy()
                assert np.array_equal(v[:n], r[k].astype(np.float32)) and not v[n:].any(), (k, b)
        else:
            assert int(out['box_num'][b]) == n and int(out['init_slot'][b]) == r['init_slot']
            got = sel[b].reshape(200, 256)
            for i in range(n):
                assert np.array_equal(got[i, :len(r['sel'][i])], r['sel'][i])
            _cmp(out['conf_points'][b].cpu(), r['conf_points'], list(range(3)) + list(range(4, 31)), [3, 31], ('c', b))
            assert np.array_equal(out['conf_score'][b].cpu().numpy(), r['conf_score'].astype(np.float32))
            assert np.array_equal(out['iou'][b].cpu().numpy(), r['iou'].astype(np.float32))


@pytest.mark.parametrize('kind', ['grm', 'crm'])
def test_training_inputs_match_oracle(cuda, seq, kind):
    s, tg, iou = seq
    frames, off, poses, tb = _dev(s, cuda)
    out = _build(kind, frames, off, poses, tb, tg, iou)
    check_against_oracle(kind, out, s, tg, iou)
    bf, bo, bp, btb = D.crop_tracks(frames, off, poses, tb)
    once = _build(kind, bf, bo, bp, btb, tg, iou, crop=False)
    for k in out:
        assert torch.equal(out[k], once[k]), k


def test_crop_tracks_is_the_crop(cuda, seq):
    """crop_tracks' rows are the in-box rows of each box's frame in frame order, and every eval builder gives the same bits on them
    with crop=False as on the original frames with crop=True"""
    s = seq[0]
    frames, off, poses, tb = _dev(s, cuda)
    bf, bo, bp, btb = D.crop_tracks(frames, off, poses, tb)
    bf, bo = bf.cpu().numpy(), bo.cpu().numpy()
    t = 0
    for b in range(len(tb)):
        for j in range(int(s['box_num'][b])):
            f = int(s['frame_of_box'][b, j])
            fr = s['frames'][s['frame_offsets'][f]:s['frame_offsets'][f + 1]]
            rows = R.crop_box(np.concatenate([fr[:, 1:4], np.arange(len(fr))[:, None]], 1), s['poses'][f], s['boxes'][b, j])
            assert np.array_equal(bf[bo[t]:bo[t + 1]], fr[rows[:, 3].astype(np.int64)]), (b, j)
            assert np.array_equal(bp[t].cpu().numpy(), s['poses'][f]) and int(btb.frame_of_box[b, j]) == t
            t += 1
    assert t == len(bo) - 1 and bo[-1] == len(bf)
    for kind, fn in (('prm', D.position_inputs), ('crm', D.confidence_inputs), ('grm', D.geometry_inputs)):
        a = fn(frames, off, poses, tb, seed=SEED, return_selection=True)
        o = fn(torch.from_numpy(bf).to(cuda), bo, bp, btb, seed=SEED, crop=False, return_selection=True)
        for k in a:
            assert torch.equal(a[k], o[k]), (kind, k)


def test_batch_order_chunks_and_repeats(cuda):
    s = synthetic.synthetic_sequence(5, frames=16, tracks=40, n_background=8000)
    tg, iou = _targets(s, cuda, seed=6)
    frames, off, poses, tb = _dev(s, cuda)
    perm = np.random.default_rng(0).permutation(len(tb))
    for kind in ('grm', 'crm'):
        a = _build(kind, frames, off, poses, tb, tg, iou)
        again = _build(kind, frames, off, poses, tb, tg, iou)
        for k in a:
            assert torch.equal(a[k], again[k]), (kind, k)
        p = _build(kind, frames, off, poses, tb.select(perm.tolist()), tg.select(perm.tolist()), iou[perm])
        parts = [(idx, _build(kind, frames, off, poses, tb.select(idx), tg.select(idx), iou[idx])) for idx in
                 (list(range(0, 7)), list(range(7, 40)))]
        for k in a:
            for rows, got in [(perm.tolist(), p)] + parts:
                want = a[k][rows]
                if kind == 'grm' and k in ('geo_query_points', 'geo_query_boxes', 'gt_geo_query_boxes'):
                    n = got[k].shape[1]
                    assert torch.equal(got[k], want[:, :n]) and not want[:, n:].any(), (kind, k)
                else:
                    assert torch.equal(got[k], want), (kind, k)
        assert not torch.equal(a['kept'], _build(kind, frames, off, poses, tb, tg, iou, epoch=EPOCH + 1)['kept']), kind


def test_rejections(cuda, seq):
    s, tg, iou = seq
    frames, off, poses, tb = _dev(s, cuda)
    bad = tg.select(list(range(len(tb))))
    bad.matched_tracklet = bad.matched_tracklet.clone()
    bad.matched_tracklet[3] = 0
    with pytest.raises(ValueError, match='matched'):
        D.geometry_training_inputs(frames, off, poses, tb, bad)
    bad = tg.select(list(range(len(tb))))
    bad.matched = bad.matched.clone()
    bad.matched[2] = 0
    with pytest.raises(ValueError, match='matched'):
        D.geometry_training_inputs(frames, off, poses, tb, bad)
    for fn, arg, base in ((D.geometry_training_inputs, tg, D.grm_train_cfg()), (D.confidence_training_inputs, iou, D.crm_train_cfg())):
        with pytest.raises(ValueError, match='AUGMENT_FULL'):
            fn(frames, off, poses, tb, arg, cfg=dict(base, AUGMENTOR={'AUGMENT_SINGLE': True, 'AUGMENT_FULL': True}))
        with pytest.raises(ValueError, match='ENCODING'):
            fn(frames, off, poses, tb, arg, cfg=dict(base, ENCODING=base['ENCODING'] + ['class']))


# ---- workspaces of the new entry points --------------------------------------------------------------------------------------
@pytest.mark.parametrize('tracks,lengths', [(10, [24, 1, 2, 17, 24, 5, 9, 24, 3, 12]), (1, [1])])
def test_workspaces(cuda, tracks, lengths):
    s = synthetic.synthetic_sequence(3, frames=24, tracks=tracks, n_background=20000, lengths=lengths)
    tg, iou = _targets(s, cuda)
    frames, foff, poses, tb = _dev(s, cuda)
    off, F, max_pts, poses = D._frames_args(frames, foff, poses)
    B, Lb = len(tb), tb.L
    W = frames.shape[1]

    cnt = D.confidence_inputs(frames, foff, poses, tb, return_selection=True)['crop_counts'].long()
    rbase = (torch.cumsum(cnt.reshape(-1), 0) - cnt.reshape(-1)).to(torch.int32).reshape(B, Lb).contiguous()
    total = int(cnt.sum())

    def crop_setup(rows_out):
        def setup():
            counts = _blank(B, Lb, dtype=torch.int32)
            rb, rows = (rbase, _blank(max(total, 1), W)) if rows_out else (None, None)
            return (lambda ws, nb: L_().dz_crop_tracks(P(frames), frames.stride(0), W, P(off), F, max_pts, P(poses), P(tb.boxes),
                                                       P(tb.frame_of_box), P(tb.box_num), B, Lb, 1.1, 0, P(counts), P(rb), P(rows), P(ws),
                                                       nb, ops._stream()),
                    [counts] + ([] if rows is None else [rows]))
        return setup
    check_workspace(L_().dz_crop_tracks_ws_bytes(B, Lb, max_pts), crop_setup(False))
    check_workspace(L_().dz_crop_tracks_ws_bytes(B, Lb, max_pts), crop_setup(True))
    for kind in (D.GRM, D.CRM):
        nq = 3 if kind == D.GRM else 1
        matched = tg.matched.contiguous()

        def draw_setup():
            o = [_blank(B, Lb, dtype=torch.int32), _blank(B, dtype=torch.int32),
                 _blank(B, nq, dtype=torch.int32) if kind == D.GRM else None, _blank(B, dtype=torch.int32) if kind == D.CRM else None,
                 _blank(B, Lb, dtype=torch.uint8) if kind == D.GRM else None]
            return (lambda ws, nb: L_().dz_refine_train_draw(kind, P(tb.box_num), P(matched), P(tb.track_uid), B, Lb, nq, SEED, EPOCH,
                                                             *[P(t) for t in o], P(ws), nb, ops._stream()), [t for t in o if t is not None])
        check_workspace(L_().dz_refine_train_draw_ws_bytes(B, Lb), draw_setup)
        cfg = D.grm_train_cfg() if kind == D.GRM else D.crm_train_cfg()
        draws = _build('grm' if kind == D.GRM else 'crm', frames, foff, poses, tb, tg, iou)
        kq, km = 256, (4096 if kind == D.GRM else 0)
        q_out = min(nq, int(draws['kept_num'].max())) if kind == D.GRM else 0

        def inputs_setup():
            if kind == D.GRM:
                o = [_blank(B, q_out, kq, 4), _blank(B, km, 11), _blank(B, Lb, 7), _blank(B, q_out, 7), _blank(B, q_out, 7),
                     _blank(B, Lb, 7), None, _blank(B, dtype=torch.int32)]
                d = [draws['kept'], draws['kept_num'], draws['query_slots'], None, draws['flip']]
                nsel = nq * kq + km
            else:
                o = [_blank(B, Lb, kq, 32), None, None, _blank(B, Lb), None, None, _blank(B, Lb), None]
                d = [draws['kept'], draws['box_num'], None, draws['init_slot'], None]
                nsel = Lb * kq
            o += [_blank(B, Lb, dtype=torch.int32), _blank(B, nsel, dtype=torch.int32)]
            call = (lambda ws, nb: L_().dz_refine_train_inputs(
                kind, P(frames), frames.stride(0), P(off), F, max_pts, P(poses), P(tb.boxes), P(tb.frame_of_box), P(tb.scores),
                P(tb.cls), P(tb.track_uid), P(tg.gt_boxes), P(iou), B, Lb, kq, km, nq, q_out, 1.1, 0, 1, SEED, EPOCH,
                *[P(t) for t in d], *[P(t) for t in o], P(ws), nb, ops._stream()))
            return call, [t for t in o if t is not None]
        assert cfg['QUERY_POINTS_NUM'] == kq
        check_workspace(L_().dz_refine_train_inputs_ws_bytes(kind, B, Lb, max_pts, kq, km, nq), inputs_setup)


# ---- end to end ------------------------------------------------------------------------------------------------------------------
def _train_model(kind):
    if kind == 'grm':
        c = ri.grm_cfg()
        c.DECODER['dropout'] = 0.0
        spec = {'NAME': 'GeometryRefineModel', 'QUERY_POINT_DIMS': 11, 'MEMORY_POINT_DIMS': 4}
    else:
        c = ri.crm_cfg()
        spec = {'NAME': 'ConfidenceRefineModel', 'QUERY_POINT_DIMS': 32, 'MEMORY_POINT_DIMS': 32}
    c.COMPUTE_MODE = 'tf32'
    m = RefineTemplate(AttrDict(dict(spec, REGRESSION=c)))
    weights.load_seeded(m.reg, SEED)
    return m.cuda().train()


def _step(kind, batch):
    m = _train_model(kind)
    ret, tb, _ = m(dict(batch))
    ret['loss'].backward()
    return {k: float(v.detach()) for k, v in tb.items()}


def test_tracked_sequence_to_training_steps(cuda):
    """track_sequences -> assign_track_target -> track_targets -> PRM and GRM eval -> revert -> refine_iou_labels -> crop_tracks ->
    training_order -> both training builders -> one tf32 training step of each model, against the same step on oracle-built
    samples"""
    s = synthetic.synthetic_sequence(7, frames=30, tracks=40, n_background=500, ego_step=0.5, max_speed=0.3, cls=[1] * 40)
    infos = synthetic.synthetic_ground_truth(s, 7, name='seq7')
    # the ground truth loses 8 of its objects, so their tracks are unmatched: the CRM's negatives
    drop = sorted({o for f in infos for o in f['annos']['obj_ids']})[:8]
    for f in infos:
        keep = ~np.isin(f['annos']['obj_ids'], drop)
        f['annos'] = {k: (v[keep] if isinstance(v, np.ndarray) and len(v) == len(keep) else v) for k, v in f['annos'].items()}
    boxes, counts, _ = synthetic.detections_from_sequence(s, 7)
    res = track_sequences(torch.from_numpy(boxes)[None].cuda(), torch.from_numpy(counts)[None], torch.from_numpy(s['poses'])[None],
                          max_entries=1 << 20)
    gt = ground_truth_from_infos(infos, ['seq7'])
    assign = assign_track_target(res, gt)
    tb = res.track_batch('Vehicle')
    tg = D.track_targets(assign, tb)
    frames, off, poses = torch.from_numpy(s['frames']).to(cuda), s['frame_offsets'], torch.from_numpy(s['poses']).to(cuda)
    models = synthetic.refine_models(7, classes=['Vehicle'])['Vehicle']
    with torch.no_grad():
        prm = models['PRM'].reg.eval()(D.position_inputs(frames, off, poses, tb))['batch_box_preds']
        grm = models['GRM'].reg.eval()(D.geometry_inputs(frames, off, poses, tb))['batch_box_preds']
    _, world = D.revert_position_boxes(prm, poses, tb)
    iou = S.refine_iou_labels(world, grm, tb, tg)
    bf, bo, bp, btb = D.crop_tracks(frames, off, poses, tb)
    host = {k: v.cpu().numpy() for k, v in (('boxes', tb.boxes), ('frame_of_box', tb.frame_of_box), ('scores', tb.scores),
                                            ('box_num', tb.box_num), ('cls', tb.cls), ('track_uid', tb.track_uid))}
    report = {}
    for kind in ('grm', 'crm'):
        order = D.training_order(tg, kind, seed=SEED, epoch=EPOCH)
        if kind == 'crm':
            assert len(order) == 2 * int(tg.matched_tracklet.sum()) and len(order) >= 8
        idx = order[:min(len(order), 16)].tolist()
        sub = {k: v[idx] for k, v in host.items()}
        if kind == 'grm':
            dev = D.geometry_training_inputs(bf, bo, bp, btb.select(idx),
                                             tg.select(idx), seed=SEED, epoch=EPOCH, crop=False)
            ref = T.build_train_batch('grm', s['frames'], s['frame_offsets'], s['poses'], sub, SEED, EPOCH,
                                      gt_boxes=tg.gt_boxes[idx].cpu().numpy(), matched=tg.matched[idx].cpu().numpy())
            Q = dev['geo_query_points'].shape[1]
            qp, qb, gq = np.zeros((len(idx), Q, 256, 4)), np.zeros((len(idx), Q, 7)), np.zeros((len(idx), Q, 7))
            for i, r in enumerate(ref):
                n = r['geo_query_num']
                qp[i, :n], qb[i, :n], gq[i, :n] = r['geo_query_points'], r['geo_query_boxes'], r['gt_geo_query_boxes']
            up = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.float32, device=cuda)  # noqa: E731
            host_batch = {'geo_query_points': up(qp), 'geo_query_boxes': up(qb), 'gt_geo_query_boxes': up(gq),
                          'geo_memory_points': up(np.stack([r['geo_memory_points'] for r in ref])),
                          'geo_query_num': torch.tensor([r['geo_query_num'] for r in ref], device=cuda)}
            a, b = _step(kind, dev), _step(kind, host_batch)
            key = 'geometry_loss'
        else:
            dev = D.confidence_training_inputs(bf, bo, bp, btb.select(idx), iou[idx], seed=SEED, epoch=EPOCH, crop=False)
            ref = T.build_train_batch('crm', s['frames'], s['frame_offsets'], s['poses'], sub, SEED, EPOCH, iou=iou[idx].cpu().numpy())
            up = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.float32, device=cuda)  # noqa: E731
            a = _step(kind, {'conf_points': dev['conf_points'], 'iou': dev['iou']})
            b = _step(kind, {'conf_points': up(np.stack([r['conf_points'] for r in ref])), 'iou': up(np.stack([r['iou'] for r in ref]))})
            key = max(a, key=lambda k: abs(a[k]))
        for k in a:
            assert np.isfinite(a[k]), (kind, k)
            assert abs(a[k] - b[k]) <= LOSS_TOL * max(abs(b[k]), 1e-6), (kind, k, a[k], b[k])
        report[kind] = (key, a[key], b[key])
    print('training step on device vs oracle samples:', report)

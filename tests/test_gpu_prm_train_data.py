"""PRM training samples built on the device (refine.data.position_training_inputs, training_order('prm'); csrc/refine_data.cu
dz_refine_train_draw kind 0 and dz_position_train_inputs) against the float64 restatement (tests/prm_train_data_ref.py) on
synthetic sequences at Waymo-like world offsets (~5 km): the keyed draws exactly, the features within test_gpu_refine_data.py's
tolerances, the crop-once path bit for bit, batch-order / chunk / repeat independence, the rejections, the workspaces of the new
entry points, and the chain from a tracked and assigned sequence to samples the PRM consumes and trains on."""
import numpy as np
import pytest
import torch

from detzero_b200 import _lib, ops, synthetic
from detzero_b200.refine import data as D
from detzero_b200.track import assign_track_target, ground_truth_from_infos, track_sequences
from tests import prm_train_data_ref as PT
from tests.test_gpu_refine_train_data import _dev, _targets
from tests.test_gpu_workspace import _blank, check_workspace

pytestmark = pytest.mark.gpu
SEED, EPOCH = 21, 4
COORD_TOL = 5e-5          # metres, columns derived from coordinates (xyz, p2co, trajectories); as test_gpu_refine_data.py
L_ = _lib.lib
P = ops._p
XYZ_P2CO = list(range(3)) + list(range(4, 31))


@pytest.fixture(scope='module')
def seq():
    s = synthetic.synthetic_sequence(3, frames=24, tracks=10, n_background=20000, lengths=[24, 1, 2, 17, 24, 5, 9, 24, 3, 12])
    tg, _ = _targets(s, 'cuda')
    return s, tg


def _build(frames, off, poses, tb, tg, crop=True, epoch=EPOCH, **kw):
    return D.position_training_inputs(frames, off, poses, tb, tg, seed=SEED, epoch=epoch, crop=crop, return_selection=True, **kw)


def check_against_oracle(out, s, tg):
    ref = PT.build_position_train_batch(s['frames'], s['frame_offsets'], s['poses'], s, SEED, EPOCH, tg.gt_boxes.cpu().numpy(),
                                        tg.matched.cpu().numpy())
    kept, counts, sel = out['kept'].cpu().numpy(), out['crop_counts'].cpu().numpy(), out['selection'].cpu().numpy()
    L = kept.shape[1]
    for b, r in enumerate(ref):
        n = r['box_num']
        assert np.array_equal(kept[b, :n], r['kept']) and (kept[b, n:] == -1).all(), b
        assert int(out['box_num'][b]) == n and int(out['init_slot'][b]) == r['init_slot'], b
        assert np.array_equal(counts[b, :n], r['counts']), b
        got = sel[b].reshape(L, 256 + 48)
        for i in range(n):
            assert np.array_equal(got[i, :len(r['sel'][0][i])], r['sel'][0][i]), (b, i)
            assert np.array_equal(got[i, 256:256 + len(r['sel'][1][i])], r['sel'][1][i]), (b, i)
        for k in ('pos_query_points', 'pos_memory_points'):
            v = out[k][b].cpu().numpy().astype(np.float64)
            assert np.abs(v[..., XYZ_P2CO] - r[k][..., XYZ_P2CO]).max() <= COORD_TOL, (k, b)
            assert np.array_equal(v[..., [3, 31]], r[k][..., [3, 31]].astype(np.float32)), (k, b)
            assert not v[n:].any(), (k, b)
        for k in ('pos_trajectory', 'gt_pos_trajectory'):
            v = out[k][b].cpu().numpy()
            assert np.abs(v - r[k]).max() <= COORD_TOL and not v[n:].any(), (k, b)
        assert np.array_equal(out['padding_mask'][b].cpu().numpy(), r['padding_mask'].astype(np.float32)), b
        assert np.array_equal(out['pos_init_box'][b].cpu().numpy(), r['pos_init_box'].astype(np.float32)), b
    return ref


def test_position_training_inputs_match_oracle(cuda, seq):
    s, tg = seq
    frames, off, poses, tb = _dev(s, cuda)
    out = _build(frames, off, poses, tb, tg)
    ref = check_against_oracle(out, s, tg)
    assert any(r['init_slot'] != r['box_num'] // 2 for r in ref) and any(r['box_num'] < s['box_num'][b] for b, r in enumerate(ref))
    bf, bo, bp, btb = D.crop_tracks(frames, off, poses, tb)
    once = _build(bf, bo, bp, btb, tg, crop=False)
    for k in out:
        assert torch.equal(out[k], once[k]), k


def test_batch_order_chunks_and_repeats(cuda):
    s = synthetic.synthetic_sequence(5, frames=16, tracks=40, n_background=8000)
    tg, _ = _targets(s, cuda, seed=6)
    frames, off, poses, tb = _dev(s, cuda)
    perm = np.random.default_rng(0).permutation(len(tb))
    a = _build(frames, off, poses, tb, tg)
    again = _build(frames, off, poses, tb, tg)
    for k in a:
        assert torch.equal(a[k], again[k]), k
    p = _build(frames, off, poses, tb.select(perm.tolist()), tg.select(perm.tolist()))
    parts = [(idx, _build(frames, off, poses, tb.select(idx), tg.select(idx))) for idx in (list(range(0, 7)), list(range(7, 40)))]
    for k in a:
        for rows, got in [(perm.tolist(), p)] + parts:
            assert torch.equal(got[k], a[k][rows]), k
    assert not torch.equal(a['kept'], _build(frames, off, poses, tb, tg, epoch=EPOCH + 1)['kept'])


def test_rejections(cuda, seq):
    s, tg = seq
    frames, off, poses, tb = _dev(s, cuda)
    bad = tg.select(list(range(len(tb))))
    bad.matched_tracklet = bad.matched_tracklet.clone()
    bad.matched_tracklet[3] = 0
    with pytest.raises(ValueError, match='matched'):
        D.position_training_inputs(frames, off, poses, tb, bad)
    bad = tg.select(list(range(len(tb))))
    bad.matched = bad.matched.clone()
    bad.matched[2] = 0
    with pytest.raises(ValueError, match='matched'):
        D.position_training_inputs(frames, off, poses, tb, bad)
    base = D.prm_train_cfg()
    with pytest.raises(ValueError, match='AUGMENT_FULL'):
        D.position_training_inputs(frames, off, poses, tb, tg, cfg=dict(base, AUGMENTOR={'AUGMENT_FULL': True}))
    for enc in (base['ENCODING'] + ['class'], ['xyz', 'intensity', 'p2s', 'score']):
        with pytest.raises(ValueError, match='ENCODING'):
            D.position_training_inputs(frames, off, poses, tb, tg, cfg=dict(base, ENCODING=enc))
    with pytest.raises(ValueError, match='MEMORY_POINTS_NUM'):
        D.position_training_inputs(frames, off, poses, tb, tg, cfg=dict(base, MEMORY_POINTS_NUM=64))
    with pytest.raises(ValueError, match='QUERY_NUM'):
        D.position_training_inputs(frames, off, poses, tb, tg, cfg=dict(base, QUERY_NUM=100))
    # the PRM draw refuses to run without its matched mask
    B, L = len(tb), tb.L
    ws = torch.empty(L_().dz_refine_train_draw_ws_bytes(B, L), dtype=torch.uint8, device=cuda)
    kept, n_kept, init = (torch.empty((B, L), dtype=torch.int32, device=cuda), torch.empty((B,), dtype=torch.int32, device=cuda),
                          torch.empty((B,), dtype=torch.int32, device=cuda))
    assert L_().dz_refine_train_draw(D.PRM, P(tb.box_num), None, P(tb.track_uid), B, L, 1, SEED, EPOCH, P(kept), P(n_kept), None,
                                     P(init), None, P(ws), ws.numel(), ops._stream()) == _lib.DZ_ERR_ARG


@pytest.mark.parametrize('tracks,lengths', [(10, [24, 1, 2, 17, 24, 5, 9, 24, 3, 12]), (1, [1])])
def test_workspaces(cuda, tracks, lengths):
    s = synthetic.synthetic_sequence(3, frames=24, tracks=tracks, n_background=20000, lengths=lengths)
    tg, _ = _targets(s, cuda)
    frames, foff, poses, tb = _dev(s, cuda)
    off, F, max_pts, poses = D._frames_args(frames, foff, poses)
    B, Lb = len(tb), tb.L
    matched = tg.matched.contiguous()

    def draw_setup():
        o = [_blank(B, Lb, dtype=torch.int32), _blank(B, dtype=torch.int32), _blank(B, dtype=torch.int32)]
        return (lambda ws, nb: L_().dz_refine_train_draw(D.PRM, P(tb.box_num), P(matched), P(tb.track_uid), B, Lb, 1, SEED, EPOCH,
                                                         P(o[0]), P(o[1]), None, P(o[2]), None, P(ws), nb, ops._stream()), o)
    check_workspace(L_().dz_refine_train_draw_ws_bytes(B, Lb), draw_setup)
    draws = _build(frames, foff, poses, tb, tg)
    kq, km = 256, 48

    def inputs_setup():
        o = [_blank(B, Lb, kq, 32), _blank(B, Lb, km, 32), _blank(B, Lb, 7), _blank(B, Lb, 7), _blank(B, Lb), _blank(B, 7),
             _blank(B, Lb, dtype=torch.int32), _blank(B, Lb * (kq + km), dtype=torch.int32)]
        call = (lambda ws, nb: L_().dz_position_train_inputs(
            P(frames), frames.stride(0), P(off), F, max_pts, P(poses), P(tb.boxes), P(tb.frame_of_box), P(tb.scores), P(tb.cls),
            P(tb.track_uid), P(tg.gt_boxes), B, Lb, kq, km, 1.1, 0, 1, SEED, EPOCH, P(draws['kept']), P(draws['box_num']),
            P(draws['init_slot']), *[P(t) for t in o], P(ws), nb, ops._stream()))
        return call, o
    check_workspace(L_().dz_position_train_inputs_ws_bytes(B, Lb, max_pts, kq, km), inputs_setup)


def test_tracked_sequence_to_position_samples(cuda):
    """track_sequences -> assign_track_target -> track_targets -> crop_tracks -> training_order('prm') -> position_training_inputs,
    against the restatement on the same tracks, and the PRM runs on the samples"""
    s = synthetic.synthetic_sequence(7, frames=30, tracks=40, n_background=500, ego_step=0.5, max_speed=0.3, cls=[1] * 40)
    infos = synthetic.synthetic_ground_truth(s, 7, name='seq7')
    drop = sorted({o for f in infos for o in f['annos']['obj_ids']})[:8]        # unmatched tracks, which the order leaves out
    for f in infos:
        keep = ~np.isin(f['annos']['obj_ids'], drop)
        f['annos'] = {k: (v[keep] if isinstance(v, np.ndarray) and len(v) == len(keep) else v) for k, v in f['annos'].items()}
    boxes, counts, _ = synthetic.detections_from_sequence(s, 7)
    res = track_sequences(torch.from_numpy(boxes)[None].cuda(), torch.from_numpy(counts)[None], torch.from_numpy(s['poses'])[None],
                          max_entries=1 << 20)
    assign = assign_track_target(res, ground_truth_from_infos(infos, ['seq7']))
    tb = res.track_batch('Vehicle')
    tg = D.track_targets(assign, tb)
    frames, off, poses = torch.from_numpy(s['frames']).to(cuda), s['frame_offsets'], torch.from_numpy(s['poses']).to(cuda)
    bf, bo, bp, btb = D.crop_tracks(frames, off, poses, tb)
    order = D.training_order(tg, 'prm', seed=SEED, epoch=EPOCH)
    mt = tg.matched_tracklet.cpu().numpy() != 0
    assert 0 < len(order) < len(tb) and mt[order].all()
    idx = order[:16].tolist()
    dev = _build(bf, bo, bp, btb.select(idx), tg.select(idx), crop=False)
    host = {k: v[idx].cpu().numpy() for k, v in (('boxes', tb.boxes), ('frame_of_box', tb.frame_of_box), ('scores', tb.scores),
                                                 ('box_num', tb.box_num), ('cls', tb.cls), ('track_uid', tb.track_uid))}
    sub = dict(s, **host)
    check_against_oracle(dev, sub, tg.select(idx))
    models = synthetic.refine_models(7, classes=['Vehicle'])['Vehicle']
    with torch.no_grad():
        pred = models['PRM'].reg.eval()({k: dev[k] for k in ('pos_query_points', 'pos_memory_points', 'pos_trajectory',
                                                               'padding_mask', 'pos_init_box', 'box_num')})['batch_box_preds']
    assert pred.shape == (len(idx), tb.L, 7) and bool(torch.isfinite(pred).all())
    # one tf32 training step on the samples: a finite loss, and every parameter with a gradient above 1e-6 moves under Adam (the
    # attention key bias's gradient is zero up to rounding, as the softmax cancels it, and Adam's eps 1e-8 scales such a step below
    # an ulp); then, with dropout
    # 0, 20 Adam steps on this one batch lower the loss
    from tests.test_gpu_prm_train import model
    for dropout, steps in ((0.1, 1), (0.0, 20)):
        m = model('tf32', dropout=dropout)
        opt = torch.optim.Adam(m.parameters(), lr=1e-3)
        before = {n: p.detach().clone() for n, p in m.named_parameters()}
        losses = []
        for _ in range(steps):
            opt.zero_grad(set_to_none=True)
            ret, tbd, _ = m(dict(dev))
            ret['loss'].backward()
            if not losses:
                with_grad = [n for n, p in m.named_parameters() if p.grad is not None and float(p.grad.abs().max()) > 1e-6]
            opt.step()
            losses.append(float(ret['loss']))
        assert all(np.isfinite(losses)), losses
        if steps == 1:
            assert len(with_grad) >= 0.9 * len(before), (len(with_grad), len(before))
            assert all(not torch.equal(before[n], dict(m.named_parameters())[n]) for n in with_grad)
        else:
            assert losses[-1] < 0.8 * losses[0], losses

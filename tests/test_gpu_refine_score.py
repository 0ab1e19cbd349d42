"""refine.data.track_targets and refine.score (csrc/refine_gt.cu) against the reference's golden vectors
(tests/golden/refine_score.npz) and the numpy restatement (oracle/refine_score_ref.py).

Integer entries must equal the golden file's, and the oracle's on the synthetic sequences wherever its decision margin is at least
1e-3.  Per-box IoUs follow the bounds tests/test_gpu_track_gt.py documents for the float32 clip: at most one box in a thousand further
than 5e-5 from the oracle, none further than 2e-2 (1e-5 on the golden scene)."""
import numpy as np
import pytest
import torch

from detzero_b200 import offboard, synthetic
from detzero_b200.refine import data as D
from detzero_b200.refine import score as S
from detzero_b200.track import (CLASS_NAMES, IoU3D_dis_mat, TrackResult, assign_track_target, ground_truth_from_infos,
                                track_sequences)
from oracle import refine_score_ref as R
from oracle import track_gt_ref
from tests import refine_score_golden as G

pytestmark = pytest.mark.gpu


def _track_result(tracks, F, poses):
    """a one-sequence TrackResult of track dicts {id: {'boxes_global', 'name', 'sample_idx', 'score', 'state'}}"""
    T, E = max(len(tracks), 1), max(sum(len(v['name']) for v in tracks.values()), 1)
    trk = np.zeros((1, T, 6), np.int32)
    eb, ef, es = np.zeros((1, E, 9)), np.zeros((1, E), np.int32), np.zeros((1, E), np.float32)
    off = 0
    for k, (tid, t) in enumerate(tracks.items()):
        c = len(t['name'])
        fr = [int(x) for x in t['sample_idx']]
        trk[0, k] = [tid, CLASS_NAMES.index(str(t['name'][0])) + 1, fr[0], c, t['state'] == 'dynamic', off]
        b = np.asarray(t['boxes_global'])
        eb[0, off:off + c, :b.shape[1]] = b[:, :9]
        ef[0, off:off + c], es[0, off:off + c] = fr, t['score']
        off += c
    d = lambda a: torch.from_numpy(a).cuda()
    return TrackResult(d(np.zeros((1, F, 1, 9), np.float32)), d(np.zeros((1, F), np.int32)), poses, d(np.full(1, F, np.int32)),
                       d(trk), d(np.array([len(tracks)], np.int32)), d(eb), d(es), d(np.ones((1, E), np.int32)), d(ef),
                       d(np.zeros((1, F, 1), np.uint8)))


@pytest.fixture(scope='module')
def golden():
    g, frames, tracks = G.load()
    gt = ground_truth_from_infos(frames, ['seq'])
    tr = _track_result(tracks, len(frames), gt.poses)
    assign = assign_track_target(tr, gt, G.ASSIGN_THR)
    assigned, _ = track_gt_ref.assign_track_target(frames, tracks, G.ASSIGN_THR)
    infos = R.attach_targets(assigned)
    return g, tr, gt, assign, {tid: infos[tid] for tid in tracks}


def _pad(rows, L, width=None, fill=0.0):
    out = np.full((len(rows), L) + ((width,) if width else ()), fill, np.float64)
    for b, r in enumerate(rows):
        out[b, :len(r)] = r
    return out


def _check_targets(tg, tb, infos):
    L = tb.L
    assert np.array_equal(tg.gt_boxes.cpu().numpy(), _pad([i['gt_boxes_global'] for i in infos.values()], L, 7))
    assert np.array_equal(tg.matched.cpu().numpy(), _pad([i['matched'] for i in infos.values()], L))
    assert tg.matched_tracklet.cpu().tolist() == [int(i['matched_tracklet']) for i in infos.values()]
    assert tg.state.cpu().tolist() == [int(i['state'] == 'dynamic') for i in infos.values()]
    # within 1e-5, or a float32 ulp where a zero box lands kilometres from the init box
    ref = _pad([R.gt_pos_trajectory(i) for i in infos.values()], L, 7)
    assert (np.abs(tg.gt_traj.cpu().numpy() - ref) <= 1e-5 + 1.2e-7 * np.abs(ref)).all()


def test_targets_golden(golden):
    g, tr, gt, assign, infos = golden
    tb = tr.track_batch()
    tg = D.track_targets(assign, tb)
    _check_targets(tg, tb, infos)
    sub = tg.select(slice(2, 5))
    assert torch.equal(sub.gt_boxes, tg.gt_boxes[2:5]) and torch.equal(sub.obj, tg.obj[2:5]) and len(sub) == 3
    with pytest.raises(ValueError, match='track_uid'):
        bad = tr.track_batch()
        bad.track_uid = bad.track_uid + 1000
        D.track_targets(assign, bad)


def _world(g, rows, infos):
    return [R.world_boxes(g['prm_pred'][b, :len(i['boxes_global'])], i['boxes_global'][len(i['boxes_global']) // 2])
            for b, i in zip(rows, infos.values())]


def _iou_close(dev, ref, tight):
    err = np.abs(np.asarray(dev, np.float64) - np.asarray(ref, np.float64))
    if tight:
        assert err.max(initial=0) < 1e-5, err.max()
    else:
        assert err.max(initial=0) < 2e-2 and (err > 5e-5).sum() <= max(1, err.size // 1000), (err.max(), (err > 5e-5).sum())


@pytest.mark.parametrize('cls', G.CLASS_NAMES)
def test_records_golden(golden, cls):
    g, tr, gt, assign, infos_all = golden
    rows = G.class_rows(g, cls)
    ids = g['tk_ids'].tolist()
    infos = {ids[b]: infos_all[ids[b]] for b in rows}
    th = G.THRESHOLDS[cls]
    tb = tr.track_batch(cls)
    assert tb.track_uid.cpu().tolist() == list(infos)
    tg = D.track_targets(assign, tb)
    prm = torch.from_numpy(g['prm_pred'][rows]).cuda()
    grm = torch.from_numpy(g['grm_pred'][rows]).cuda()
    _, world = D.revert_position_boxes(prm, gt.poses[0], tb)
    rec = S.position_recall(world, tb, tg, th)
    ref = G.record(g, 'PRM', cls)
    assert list(rec) == list(ref) and rec == ref, {k: (rec[k], ref[k]) for k in rec if rec[k] != ref[k]}
    rec = S.geometry_recall(grm, tb, tg, th)
    ref = G.record(g, 'GRM', cls)
    assert list(rec) == list(ref) and rec == ref, {k: (rec[k], ref[k]) for k in rec if rec[k] != ref[k]}
    assert S.summarize(rec, th)['Recall@box/input_%s' % th[0]] == ref['Box level input %s' % th[0]] / max(ref['Box num'], 1)
    with pytest.raises(ValueError, match='CENTER_ALIGN'):
        S.geometry_recall(grm, tb, tg, th, center_align=True)
    # per-box IoUs against the oracle, and the labels
    iou_in, iou_out, cnt = S.score_boxes(tb.boxes, world, None, tb, tg, th)
    _, ious, _ = R.position_recall(infos, _world(g, rows, infos), th)
    for b, (info, io) in enumerate(zip(infos.values(), ious)):
        n = len(info['boxes_global'])
        if io is None:
            assert not iou_in[b].any() and not iou_out[b].any() and not cnt[b].any()
            continue
        m = info['matched']
        _iou_close(iou_in[b, :n].cpu().numpy()[m], io[0], True)
        _iou_close(iou_out[b, :n].cpu().numpy()[m], io[1], True)
        assert not iou_in[b, :n].cpu().numpy()[~m].any() and not iou_in[b, n:].any()
    lab = S.refine_iou_labels(world, grm, tb, tg)
    ref_lab = G.labels(g)
    _, comb, _ = S.score_boxes(tb.boxes, world, grm, tb, tg, th)
    for b, (r, info) in enumerate(zip(rows, infos.values())):
        n = len(info['boxes_global'])
        assert (lab[b, n:] == -1).all() and not torch.isnan(lab[b]).any()
        assert np.abs(lab[b, :n].cpu().numpy() - ref_lab[r]).max() < 2e-3      # the reference clips float32 boxes 5 km out
        m = torch.from_numpy(info['matched']).cuda()
        if info['matched_tracklet']:
            assert torch.equal(lab[b, :n][m], comb[b, :n][m]) and not lab[b, :n][~m].any()
        else:
            assert not lab[b, :n].any()                                       # against a zero box: 0, not NaN
    crm_pred = torch.from_numpy(g['crm_pred'][rows]).cuda()
    ref_iou = torch.from_numpy(_pad([ref_lab[r] for r in rows], tb.L, fill=-1).astype(np.float32)).cuda()
    rec = S.confidence_recall(tb.scores, crm_pred, ref_iou, tb, tg, th)
    ref = G.record(g, 'CRM', cls)
    assert list(rec) == g['CRM_%s_all_keys' % cls].tolist()
    assert {k: v for k, v in rec.items() if not isinstance(v, list)} == ref
    for k in ('gt_score', 'pred_score', 'ori_score'):
        assert np.array_equal(np.asarray(rec[k]), g['CRM_%s_%s' % (cls, k)]), k
    both = S.accumulate(rec, rec)
    assert both['Box num'] == 2 * rec['Box num'] and len(both['gt_score']) == 2 * len(rec['gt_score']) and list(both) == list(rec)
    assert S.accumulate({}, rec) == rec


def test_gt_traj_transform_is_position_inputs(golden):
    """the ground truth put equal to the track's own boxes: gt_traj must be pos_trajectory, bit for bit"""
    s = synthetic.synthetic_sequence(3, frames=30, tracks=6, n_background=500)
    tb = D.TrackBatch(s['boxes'], s['frame_of_box'], s['scores'], s['box_num'], s['cls'], s['track_uid'])
    B, F = len(tb), len(s['poses'])
    world = torch.zeros((F, B, 9), dtype=torch.float64, device='cuda')
    valid = torch.arange(tb.L, device='cuda')[None, :] < tb.box_num[:, None]
    bi = torch.arange(B, device='cuda')[:, None].expand(B, tb.L)
    world[tb.frame_of_box.long()[valid], bi[valid], :7] = tb.boxes[valid]
    obj = torch.arange(B, dtype=torch.int32, device='cuda')[None, :].expand(F, B)
    zero = torch.zeros(B, dtype=torch.int32)
    tg = D.refine_targets(world, obj, torch.full((F,), B, dtype=torch.int32), torch.arange(B), zero, zero, tb)
    pin = D.position_inputs(torch.from_numpy(s['frames']).cuda(), s['frame_offsets'], torch.from_numpy(s['poses']).cuda(), tb)
    assert torch.equal(tg.gt_traj, pin['pos_trajectory'])
    assert torch.equal(tg.gt_boxes[valid], tb.boxes[valid]) and bool(tg.matched[valid].all()) and not tg.matched[~valid].any()


def test_aligned_iou_is_the_diagonal():
    g = torch.Generator().manual_seed(5)
    a = torch.rand((300, 9), generator=g) * torch.tensor([20, 20, 2, 4, 2, 1.5, 6.3, 1, 1]) + torch.tensor([0, 0, 0, 0.5, 0.5, 0.5, -3.15, 0, 0])
    b = a[:, :7].clone() + torch.randn((300, 7), generator=g) * 0.2
    a, b = a.cuda(), b.cuda().contiguous()
    out = S.boxes_iou3d_aligned(a, b)
    assert torch.equal(out, IoU3D_dis_mat(a, b).diag()) and float(out.max()) > 0.3
    assert S.boxes_iou3d_aligned(a[:0], b[:0]).shape == (0,)


def _scene(seed, frames=40, objects=30, cls=None):
    s = synthetic.synthetic_sequence(seed, frames=frames, tracks=objects, n_background=500, ego_step=0.5, max_speed=0.3, cls=cls)
    infos = synthetic.synthetic_ground_truth(s, seed, name='seq%d' % seed)
    boxes, counts, _ = synthetic.detections_from_sequence(s, seed)
    res = track_sequences(torch.from_numpy(boxes)[None].cuda(), torch.from_numpy(counts)[None], torch.from_numpy(s['poses'])[None],
                          max_entries=1 << 20)
    gt = ground_truth_from_infos(infos, ['seq%d' % seed])
    return s, infos, res, gt


@pytest.mark.parametrize('seed', [1, 3])
def test_seeded_scene_vs_oracle(seed):
    s, infos, res, gt = _scene(seed)
    name = 'seq%d' % seed
    assign = assign_track_target(res, gt)
    tracks, _ = res.to_reference([name], gt.frame_ids)
    assigned, _ = track_gt_ref.assign_track_target(infos, tracks[name], {'Vehicle': 0.3, 'Pedestrian': 0.1, 'Cyclist': 0.1})
    infos_all = R.attach_targets(assigned)
    rng = np.random.default_rng(seed)
    err_c, err_u = [], []
    for cls in CLASS_NAMES:
        tb = res.track_batch(cls)
        ids = tb.track_uid.cpu().tolist()
        ti = {t: infos_all[t] for t in ids}
        tg = D.track_targets(assign, tb)
        _check_targets(tg, tb, ti)
        th = [0.7, 0.5, 0.3]
        n = [len(i['boxes_global']) for i in ti.values()]
        pred = [np.where(i['matched'][:, None] & i['matched_tracklet'], i['gt_boxes_global'], i['boxes_global'])
                + rng.normal(0, 0.05, (k, 7)) for i, k in zip(ti.values(), n)]
        grm = np.stack([np.r_[0, 0, 0, i['boxes_global'][0, 3:6] * rng.uniform(0.9, 1.1, 3), 0] for i in ti.values()]).astype(np.float32) \
            if ids else np.zeros((0, 7), np.float32)
        world = torch.from_numpy(_pad(pred, tb.L, 7)).cuda()
        ref_p, ious, m_p = R.position_recall(ti, pred, th)
        ref_g, _, m_g = R.geometry_recall(ti, grm, th)
        if min(m_p['iou'].value, m_p['ratio'].value) >= 1e-3:
            assert S.position_recall(world, tb, tg, th) == ref_p
        if min(m_g['iou'].value, m_g['ratio'].value) >= 1e-3:
            assert S.geometry_recall(torch.from_numpy(grm).cuda(), tb, tg, th) == ref_g
        iou_in, iou_out, _ = S.score_boxes(tb.boxes, world, None, tb, tg, th)
        for b, (i, io) in enumerate(zip(ti.values(), ious)):
            if io is None:
                continue
            m = i['matched']
            dev = np.concatenate([iou_in[b, :n[b]].cpu().numpy()[m], iou_out[b, :n[b]].cpu().numpy()[m]])
            err_c.append(np.abs(dev - np.concatenate(io)))
            # the same pairs clipped where they stand, 5 km from the origin
            un = np.concatenate([S.boxes_iou3d_aligned(torch.from_numpy(x[m]).float().cuda(),
                                                       torch.from_numpy(i['gt_boxes_global'][m]).float().cuda()).cpu().numpy()
                                 for x in (i['boxes_global'], pred[b])])
            err_u.append(np.abs(un - np.concatenate(io)))
        lab = S.refine_iou_labels(world, torch.from_numpy(grm).cuda(), tb, tg).cpu().numpy()
        ref_lab = R.refine_iou_labels(ti, pred, grm)
        for b in range(len(ids)):
            assert (lab[b, n[b]:] == -1).all()
            _iou_close(lab[b, :n[b]], ref_lab[b], False)
    err_c, err_u = np.concatenate(err_c), np.concatenate(err_u)
    _iou_close(err_c, 0 * err_c, False)
    assert len(err_c) > 500 and err_c.mean() <= err_u.mean() and err_c.max() <= max(err_u.max(), 5e-5)


@pytest.fixture(scope='module')
def offboard_scene():
    s, infos, res, gt = _scene(7, frames=30, objects=40)
    models = synthetic.refine_models(7)
    args = (torch.from_numpy(s['frames']).cuda(), s['frame_offsets'], torch.from_numpy(s['poses']).cuda(), res, models)
    return args, assign_track_target(res, gt), gt


def test_refine_sequence_scored(offboard_scene):
    args, assign, gt = offboard_scene
    with torch.no_grad():
        plain = offboard.refine_sequence(*args, chunk=16)
        timings = {}
        a = offboard.refine_sequence(*args, chunk=16, assign=assign, timings=timings)
        b = offboard.refine_sequence(*args, chunk=64, assign=assign)
        a2 = offboard.refine_sequence(*args, chunk=16, assign=assign)
    assert plain.recall is None and 'refine_iou' not in plain.tables
    assert {'targets', 'score'} <= set(timings)
    for r in (a, b):
        assert torch.equal(r.rows, plain.rows) and torch.equal(r.obj_id, plain.obj_id) and torch.equal(r.count, plain.count)
    assert set(a.recall) == set(CLASS_NAMES) and set(a.recall['Vehicle']) == {'PRM', 'GRM', 'CRM'}
    assert a.recall == b.recall                                              # the sum over chunks is the unchunked record
    assert a.recall == a2.recall and torch.equal(a.tables['refine_iou'], a2.tables['refine_iou'])
    assert torch.equal(a.tables['refine_iou'], b.tables['refine_iou']) and torch.equal(a.tables['matched'], b.tables['matched'])
    B = len(a.tables['box_num'])
    assert a.tables['refine_iou'].shape == (B, 200) and a.tables['matched'].dtype == torch.uint8
    assert sum(a.recall[c]['CRM']['Box num'] for c in CLASS_NAMES) == int(a.tables['box_num'].sum())
    assert sum(a.recall[c]['PRM']['Track num'] for c in CLASS_NAMES) == len(assign.matches(0)) > 0
    assert list(a.recall['Vehicle']['PRM']) == list(S.empty_record([0.7]))
    c = offboard.refine_sequence(*args, chunk=64, assign=assign, recall_thresholds={'Vehicle': [0.5, 0.3]}, combine_conf_res=False)
    assert 'Box level input 0.3' in c.recall['Vehicle']['GRM'] and set(c.recall['Vehicle']) == {'PRM', 'GRM'}


def test_empty_inputs(offboard_scene):
    args, assign, gt = offboard_scene
    res = args[3]
    tb = res.track_batch('Vehicle').select(slice(0, 0))
    tg = D.track_targets(assign, tb)
    assert len(tg) == 0 and tg.gt_boxes.shape == (0, 200, 7)
    z = torch.zeros((0, 200, 7), dtype=torch.float64, device='cuda')
    assert S.position_recall(z, tb, tg, [0.7]) == S.empty_record([0.7])
    assert S.geometry_recall(torch.zeros((0, 7), device='cuda'), tb, tg, [0.7, 0.5]) == S.empty_record([0.7, 0.5])
    lab = S.refine_iou_labels(z, torch.zeros((0, 7), device='cuda'), tb, tg)
    assert lab.shape == (0, 200)
    assert S.confidence_recall(lab, lab, lab, tb, tg, [0.5]) == S.empty_record([0.5], confidence=True)
    # a class without a track, and a sequence without ground truth
    s, _, vres, vgt = _scene(9, frames=12, objects=5, cls=[1] * 5)
    with torch.no_grad():
        only = offboard.refine_sequence(torch.from_numpy(s['frames']).cuda(), s['frame_offsets'], torch.from_numpy(s['poses']).cuda(),
                                        vres, args[4], assign=assign_track_target(vres, vgt))
    assert only.recall['Pedestrian'] == {'PRM': S.empty_record([0.5]), 'GRM': S.empty_record([0.5]),
                                         'CRM': S.empty_record([0.5], confidence=True)}
    assert only.recall['Vehicle']['PRM']['Track num'] > 0
    empty = [{'sequence_name': 'e', 'sample_idx': f, 'pose': np.eye(4),
              'annos': {'name': np.array([], '<U10'), 'obj_ids': np.array([], '<U4'), 'gt_boxes_lidar': np.zeros((0, 7), np.float32),
                        'gt_boxes_global': np.zeros((0, 9)), 'difficulty': np.zeros(0, np.int32),
                        'num_points_in_gt': np.zeros(0, np.int32)}} for f in range(int(res.num_frames[0]))]
    gt0 = ground_truth_from_infos(empty, ['e'])
    a0 = assign_track_target(res, gt0)
    tb = res.track_batch('Vehicle')
    tg = D.track_targets(a0, tb)
    assert not tg.matched_tracklet.any() and not tg.gt_boxes.any()
    assert torch.equal(tg.matched, (torch.arange(200, device='cuda')[None, :] < tb.box_num[:, None]).to(torch.uint8))
    rec = S.position_recall(tb.boxes, tb, tg, [0.7])
    assert rec == S.empty_record([0.7])
    assert not S.refine_iou_labels(tb.boxes, tb.boxes[:, 0], tb, tg).clamp_(min=0).any()

"""refine.data.combine_frames (csrc/combine.cu) and offboard.refine_sequence: the device's per-frame result against the reference's
own combine_final (tests/golden/combine.npz) and against the numpy restatement (oracle/combine_ref.py), exactly; the end-to-end
chain from ground truth through the tracker and the three refiners to the final frames."""
import numpy as np
import pytest
import torch

from detzero_b200 import offboard, synthetic
from detzero_b200.refine import data as rdata
from detzero_b200.track import CLASS_NAMES, track_sequences
from oracle import combine_ref
from tests import combine_golden as cg

pytestmark = pytest.mark.gpu
TABLE_KEYS = ('prm_lidar', 'grm_pred', 'scores', 'frame_of_box', 'box_num', 'cls', 'track_id')


def _cuda(t):
    return {k: torch.as_tensor(v).cuda() for k, v in t.items()}


def _combine(t, F, drop=None, max_rows=1024):
    """combine_frames on numpy / device tables -> OffboardResult"""
    d = _cuda({k: t[k] for k in TABLE_KEYS})
    rows, oid, cnt = rdata.combine_frames(*[d[k] for k in TABLE_KEYS], F, drop=drop, max_rows=max_rows)
    return offboard.OffboardResult(d, torch.as_tensor(t['poses']), rows, oid, cnt)


@pytest.mark.parametrize('variant', list(cg.VARIANTS))
def test_device_vs_reference_golden(variant):
    g = cg.load()
    conf, with_drop = cg.VARIANTS[variant]
    got = []
    for s, name in enumerate(cg.SEQS):
        t = cg.tables(g, s)
        if conf:
            t['scores'] = t['crm']
        drop = tuple(torch.as_tensor(g['s%d_%s' % (s, k)]).cuda() for k in ('det', 'counts', 'kept')) if with_drop else None
        got += _combine(t, len(t['poses']), drop).to_reference(name, t['frame_ids'])
    combine_ref.assert_frames_equal(got, cg.expected(g, variant))


def _random_tables(seed, B=300, F=199, L=200, K=500):
    """B tracks of 1..199 boxes over F frames: most on consecutive frames, some in shuffled order, some with two boxes in one frame;
    drop rows of up to K per frame, a few frames without any detection"""
    g = np.random.default_rng(seed)
    n = g.integers(1, F + 1, B)
    fob = np.zeros((B, L), np.int32)
    for b in range(B):
        start = int(g.integers(0, F - n[b] + 1))
        fr = np.arange(start, start + n[b])
        if b % 17 == 3:
            fr = g.permutation(fr)
        if b % 23 == 5 and n[b] > 3:
            fr[int(g.integers(1, n[b]))] = fr[0]
        fob[b, :n[b]] = fr
    t = {'prm_lidar': np.concatenate([g.uniform(-80, 80, (B, L, 3)), g.uniform(0.5, 5, (B, L, 3)), g.uniform(-7, 7, (B, L, 1))], 2),
         'grm_pred': g.normal(0, 3, (B, 7)).astype(np.float32), 'scores': g.uniform(0, 1, (B, L)).astype(np.float32),
         'frame_of_box': fob, 'box_num': n.astype(np.int32), 'cls': g.integers(1, 4, B).astype(np.int32),
         'track_id': g.permutation(100000)[:B].astype(np.int64), 'poses': g.normal(0, 1, (F, 4, 4)), 'frame_ids': 10 * np.arange(F) + 1}
    counts = g.integers(0, K + 1, F).astype(np.int32)
    counts[g.integers(0, F, 5)] = 0
    counts[:2] = K
    det = np.zeros((F, K, 9), np.float32)
    det[..., :7] = g.uniform(-20, 20, (F, K, 7))
    det[..., 7], det[..., 8] = g.uniform(0, 1, (F, K)), g.integers(1, 4, (F, K))
    kept = g.random((F, K)) < 0.3
    return t, (det, counts, kept)


def _drop_cuda(drop):
    return tuple(torch.as_tensor(a).cuda() for a in drop)


def test_full_scale_vs_oracle_and_bit_equal_runs():
    t, drop = _random_tables(5)
    F = len(t['poses'])
    res = _combine(t, F, _drop_cuda(drop))
    dd = cg.det_drop_from_rows(*drop, t['poses'], 'seq', t['frame_ids'])       # frames without detections have no entry
    want = combine_ref.frame_list(*[t[k] for k in TABLE_KEYS], t['poses'], 'seq', t['frame_ids'], dd)
    combine_ref.assert_frames_equal(res.to_reference('seq', t['frame_ids']), want)
    assert int(res.count.max()) > 500
    again = _combine(t, F, _drop_cuda(drop))
    for a, b in ((res.rows, again.rows), (res.obj_id, again.obj_id), (res.count, again.count)):
        assert torch.equal(a, b)
    no_drop = _combine(t, F)
    combine_ref.assert_frames_equal(no_drop.to_reference('seq', t['frame_ids']),
                                    combine_ref.frame_list(*[t[k] for k in TABLE_KEYS], t['poses'], 'seq', t['frame_ids']))


def test_overflow_and_bad_frames_raise():
    t, drop = _random_tables(6, B=40, F=30)
    with pytest.raises(RuntimeError, match='max_rows'):
        _combine(t, 30, _drop_cuda(drop), max_rows=8)
    t['frame_of_box'][3, 0] = 30
    with pytest.raises(ValueError, match='frame_of_box'):
        _combine(t, 30)
    t['frame_of_box'][3, 0] = 0
    t['track_id'][0] = 1 << 31
    with pytest.raises(ValueError, match='track ids'):
        _combine(t, 30)


def test_no_tracks_gives_no_rows():
    t, drop = _random_tables(7, B=0, F=20)
    res = _combine(t, 20, _drop_cuda(drop))
    assert int(res.count.sum()) == 0 and res.to_reference('seq', t['frame_ids']) == []


def test_grm_size_equals_reverted_geometry_boxes():
    s = synthetic.synthetic_sequence(3, frames=20, tracks=8, n_background=500)
    tb = rdata.TrackBatch(s['boxes'], s['frame_of_box'], s['scores'], s['box_num'], s['cls'], s['track_uid'])
    poses = torch.from_numpy(s['poses']).cuda()
    pred = torch.from_numpy(np.random.default_rng(3).normal(0, 2, (len(tb), 7)).astype(np.float32)).cuda()
    geo = rdata.revert_geometry_boxes(pred, poses, tb)[0]
    valid = torch.arange(tb.L, device='cuda')[None] < tb.box_num[:, None].long()
    size = pred[:, None, 3:6].double().expand(-1, tb.L, -1)
    assert torch.equal(geo[..., 3:6][valid], size[valid])
    prm = rdata.revert_position_boxes(torch.zeros((len(tb), tb.L, 7), device='cuda'), poses, tb)[0]
    rows, oid, cnt = rdata.combine_frames(prm, pred, tb.scores, tb.frame_of_box, tb.box_num, tb.cls, tb.track_uid, 20)
    r = rows.cpu().numpy()
    for b in range(len(tb)):
        for j in range(int(s['box_num'][b])):
            f = int(s['frame_of_box'][b, j])
            i = int(np.flatnonzero(oid[f].cpu().numpy() == int(s['track_uid'][b]))[0])
            assert r[f, i, 3:6].tobytes() == geo[b, j, 3:6].float().cpu().numpy().tobytes()


def _scene(seed, F=40, tracks=12, cls=None):
    lengths = [int(x) for x in np.random.default_rng(seed).integers(8, F + 1, tracks)]
    s = synthetic.synthetic_sequence(seed, frames=F, tracks=tracks, n_background=2000, ego_step=0.0, max_speed=0.3, lengths=lengths,
                                     cls=cls)
    boxes, counts, gt = synthetic.detections_from_sequence(s, seed)
    for f in [f for f in range(F) if (gt[f] >= 0).any()][::8]:          # a weaker copy 5 cm away: the overlap filter drops it
        i, n = int(np.flatnonzero(gt[f] >= 0)[0]), counts[f]
        boxes[f, n] = boxes[f, i]
        boxes[f, n, 1] += 0.05
        boxes[f, n, 7] *= 0.8
        counts[f] += 1
    return s, boxes, counts


def _by_hand(s, res, models, classes, conf, drop, chunk, seq=0, seed=0):
    """the chain of refine_sequence with the public functions and the oracle's combine"""
    frames, poses = torch.from_numpy(s['frames']).cuda(), torch.from_numpy(s['poses']).cuda()
    tabs = {k: [] for k in TABLE_KEYS}
    for c in classes:
        tb = res.track_batch(c, sequence=seq)
        for c0 in range(0, len(tb), chunk):
            sub = tb.select(slice(c0, c0 + chunk))
            pred = models[c]['PRM'](rdata.position_inputs(frames, s['frame_offsets'], poses, sub, seed=seed))[0]['pred_boxes']
            size = models[c]['GRM'](rdata.geometry_inputs(frames, s['frame_offsets'], poses, sub, seed=seed))[0]['pred_boxes']
            score = (models[c]['CRM'](rdata.confidence_inputs(frames, s['frame_offsets'], poses, sub, seed=seed))[0]['pred_score']
                     if conf else sub.scores)
            lidar = rdata.revert_position_boxes(pred, poses, sub)[0]
            for k, v in zip(TABLE_KEYS, (lidar, size, score, sub.frame_of_box, sub.box_num, sub.cls, sub.track_uid)):
                tabs[k].append(v.cpu().numpy())
    t = {k: np.concatenate(v) for k, v in tabs.items()}
    F = len(s['poses'])
    fids = [str(f) for f in range(F)]
    dd = res.to_reference(['seq'], [fids])[1]['seq'] if drop else None
    return combine_ref.frame_list(*[t[k] for k in TABLE_KEYS], s['poses'], 'seq', range(F), dd)


def test_end_to_end_ground_truth_to_final_frames():
    """synthetic_sequence ground truth -> jittered detections -> track_sequences -> refine_sequence: equals the same chain by hand,
    one row per live track per frame plus the frame's dropped rows, chunking does not change a bit, combine_conf_res=False gives
    the tracker scores, a class subset leaves out the other classes"""
    seed = 4
    s, boxes, counts = _scene(seed, cls=[1, 2, 1, 2, 1, 2, 2, 1, 1, 2, 1, 2])            # no cyclist track
    F = len(s['poses'])
    empty = np.zeros_like(boxes)
    res = track_sequences(torch.from_numpy(np.stack([boxes, empty])).cuda(), torch.from_numpy(np.stack([counts, counts * 0])),
                          torch.from_numpy(np.stack([s['poses']] * 2)))
    assert int(res.n_tracks[0]) >= 12 and int(res.n_tracks[1]) == 0
    models = synthetic.refine_models(seed)
    frames, poses = torch.from_numpy(s['frames']).cuda(), torch.from_numpy(s['poses']).cuda()
    run = lambda **kw: offboard.refine_sequence(frames, s['frame_offsets'], poses, res, models, **kw)     # noqa: E731
    out = run(chunk=16)
    got = out.to_reference('seq', range(F))
    combine_ref.assert_frames_equal(got, _by_hand(s, res, models, CLASS_NAMES, True, True, 16))
    # one row per track alive in the frame, then the frame's dropped detections
    ef = res.ent_frame[0].cpu().numpy()
    alive = np.zeros(F, int)
    for tid, cls, first, cnt, dyn, off in res.tracks(0):
        alive[np.unique(ef[off:off + cnt])] += 1
    kept = res.kept[0].cpu().numpy()
    n_drop = np.array([int((~kept[f, :counts[f]]).sum()) for f in range(F)])
    assert np.array_equal(out.count.cpu().numpy(), np.where(alive > 0, alive + n_drop, 0))
    assert n_drop.sum() > 0
    # chunking
    one = run(chunk=1)
    assert torch.equal(one.rows, out.rows) and torch.equal(one.obj_id, out.obj_id)
    # tracker scores without CRM
    nc = run(combine_conf_res=False, combine_drop=False)
    combine_ref.assert_frames_equal(nc.to_reference('seq', range(F)), _by_hand(s, res, models, CLASS_NAMES, False, False, 16))
    tb = res.track_batch()
    assert torch.equal(nc.tables['scores'].sort(0).values, tb.scores.sort(0).values)
    assert int(nc.count.sum()) == int(alive.sum())
    # a class subset; CRM not needed without combine_conf_res
    ped = run(class_names=('Pedestrian',), combine_drop=False, chunk=5)
    ped_ids = {int(r[0]) for r in res.tracks(0) if r[1] == 2}
    ids = set(ped.obj_id[ped.obj_id >= 0].cpu().tolist())
    assert ids == ped_ids and set(ped.rows[..., 8][ped.obj_id >= 0].cpu().tolist()) == {2.0}
    no_crm = {c: {k: m[k] for k in ('PRM', 'GRM')} for c, m in models.items()}
    offboard.refine_sequence(frames, s['frame_offsets'], poses, res, no_crm, combine_conf_res=False)
    with pytest.raises(KeyError, match='CRM'):
        offboard.refine_sequence(frames, s['frame_offsets'], poses, res, no_crm)
    # a sequence without tracks
    assert offboard.refine_sequence(frames, s['frame_offsets'], poses, res, models, sequence=1).to_reference('empty', range(F)) == []

"""Float64 numpy restatement of the refiner training samples (detzero_b200/csrc/refine_data.cu dz_refine_train_draw /
dz_refine_train_inputs, detzero_b200/refine/data.py geometry_training_inputs / confidence_training_inputs): the training branch of
WaymoGeometryDataset / WaymoConfidenceDataset.extract_track_feature (refining/detzero_refine/datasets/waymo/), with
geometry_augment.augment_single_box (traj=None) for the GRM.  It reuses the eval restatement of oracle/refine_data_ref.py: the crop
(track_crops), the keyed sampler (sample_ranks, key_base), the p2co encoding and the init-box transform.

Deliberate deviations from the reference, besides those of refine_data_ref.py:
  5. Every random.sample / random.randint / np.random.choice / np.random.randint / np.random.random of the training branch is a
     keyed draw on (epoch_seed(seed, epoch), track_uid) (train_draw), and the point samples of a training build key on
     epoch_seed(seed, epoch) too.  So a sample depends on (seed, epoch, track_uid) only.
  6. The kept boxes stay in ascending slot order where the reference keeps random.sample's order.  Every consumer is invariant to
     the order of a track's boxes (per-box encoders, max-pools, BatchNorm statistics, decoder attention over the memory, summed
     losses), so no distribution the model sees changes.
"""
import numpy as np

from .refine_data_ref import (CRM_Q, GRM_M, GRM_Q, M64, _pad, encode_p2co, init_frame, key_base, mix64, mix64_int,
                              rz, sample_ranks, track_crops)


def init_frame_at(boxes, L, at):
    """init_frame with the init box boxes[at] (the CRM's drawn init box) in place of boxes[L // 2]: the same transform, applied to
    the trajectory re-ordered so that the drawn box sits at L // 2, then put back in slot order"""
    order = np.arange(L)
    order[[at, L // 2]] = order[[L // 2, at]]
    init, R, traj = init_frame(boxes[order], L)
    return init, R, traj[np.argsort(order)]


# ---- training samples (the training branch of WaymoGeometryDataset / WaymoConfidenceDataset.extract_track_feature) --------------
ST_TR_COUNT, ST_TR_KEEP, ST_TR_QUERY, ST_TR_INIT, ST_TR_FLIP = 5, 6, 7, 8, 9
ST_ORDER, ST_NEG = 10, 11


def epoch_seed(seed, epoch):
    """mix64(mix64(seed) + epoch) mod 2^64: the seed of one epoch's draws and point samples"""
    return mix64_int((mix64_int(int(seed) & M64) + int(epoch)) & M64)


def train_draw(kind, eligible, uid, seed, epoch, nq=3):
    """the keyed draws of one track.  eligible: its eligible slots, ascending (GRM: the matched ones, CRM: 0..L-1).
    kept count n = lo + key mod (m - lo + 1), lo = min(5, m) (random.randint(min(5, m), m)); kept slots: the k-subset rule of
    sample_ranks over the eligible ranks (random.sample); GRM: min(nq, n) query positions among the kept (np.random.choice without
    replacement) and one flip bit per kept position (np.random.random() < 0.5); CRM: the init position, key mod n
    (np.random.randint(0, n))"""
    es = epoch_seed(seed, epoch)
    eligible = np.asarray(eligible, np.int64)
    m = len(eligible)
    lo = min(5, m)
    n = lo + mix64_int(key_base(es, uid, 0, ST_TR_COUNT)) % (m - lo + 1) if m else 0
    out = {'seed': es, 'kept': eligible[sample_ranks(m, n, es, uid, 0, ST_TR_KEEP)]}
    if kind == 'grm':
        out['query'] = sample_ranks(n, min(nq, n), es, uid, 0, ST_TR_QUERY)
        with np.errstate(over='ignore'):
            keys = mix64(np.uint64(key_base(es, uid, 0, ST_TR_FLIP)) + np.arange(n, dtype=np.uint64))
        out['flip'] = (keys >> np.uint64(63)).astype(np.uint8)
    else:
        out['init'] = mix64_int(key_base(es, uid, 0, ST_TR_INIT)) % n if n else 0
    return out


def geometry_train_track(crops, boxes, scores, gt_boxes, matched, L, uid, seed, epoch, nq=3, kq=256, km=4096, augment_single=True):
    """WaymoGeometryDataset.extract_track_feature (training, augment_single_box on) for one track; crops = track_crops(...)"""
    d = train_draw('grm', np.nonzero(np.asarray(matched[:L]) != 0)[0], uid, seed, epoch, nq)
    es, kept, qidx = d['seed'], d['kept'], d['query']
    flip = d['flip'] if augment_single else np.zeros(len(kept), np.uint8)
    bx, sc, gt = boxes[kept], np.asarray(scores)[kept], np.asarray(gt_boxes, np.float64)[kept]
    local, enc = [], []
    for i, j in enumerate(kept):
        p = crops[j].copy()
        p[:, :3] = p[:, :3] @ rz(-bx[i, 6]).T
        local.append(p)
        f = p.copy()
        if flip[i]:
            f[:, 1] = -f[:, 1]                                   # augment_single_box(traj=None): after the query points are copied
        h = bx[i, 3:6] / 2
        enc.append(np.concatenate([f[:, :3], f[:, 3:4], h - f[:, :3], h + f[:, :3], np.full((len(f), 1), sc[i])], 1))
    allp = np.concatenate(enc, 0) if enc else np.zeros((0, 11))
    sm = sample_ranks(len(allp), km, es, uid, 0, GRM_M)
    qp, qb, gqb = np.zeros((len(qidx), kq, 4)), np.zeros((len(qidx), 7)), np.zeros((len(qidx), 7))
    sel_q = []
    for i, j in enumerate(qidx):
        s = sample_ranks(len(local[j]), kq, es, uid, j, GRM_Q)
        sel_q.append(s)
        qp[i] = _pad(local[j][s], kq)
        qb[i, 3:6], gqb[i, 3:6] = bx[j, 3:6], gt[j, 3:6]
    return {'geo_query_points': qp, 'geo_query_boxes': qb, 'gt_geo_query_boxes': gqb, 'geo_memory_points': _pad(allp[sm], km),
            'geo_query_num': len(qidx), 'geo_trajectory': bx, 'gt_geo_trajectory': gt, 'kept': kept, 'query_slots': qidx,
            'flip': flip, 'sel': (sel_q, sm), 'counts': np.array([len(crops[j]) for j in kept])}


def confidence_train_track(crops, boxes, scores, iou, L, uid, seed, epoch, Lmax=200, kq=256):
    """WaymoConfidenceDataset.extract_track_feature (training) for one track"""
    d = train_draw('crm', np.arange(L), uid, seed, epoch)
    es, kept, at = d['seed'], d['kept'], d['init']
    n = len(kept)
    bx, sc = boxes[kept], np.asarray(scores)[kept]
    init, R, traj = init_frame_at(bx, n, at)
    q = np.zeros((Lmax, kq, 32))
    sel = []
    for i, j in enumerate(kept):
        local = crops[j].copy()
        local[:, :3] = (local[:, :3] + (bx[i, :3] - init[:3])) @ R.T
        s = sample_ranks(len(local), kq, es, uid, i, CRM_Q)
        sel.append(s)
        q[i] = encode_p2co(_pad(local[s], kq), traj[i], sc[i], None)
    cs, io = np.full(Lmax, -1.0), np.full(Lmax, -1.0)
    cs[:n], io[:n] = sc, np.asarray(iou, np.float64)[kept]
    return {'conf_points': q, 'conf_score': cs, 'iou': io, 'box_num': n, 'kept': kept, 'init_slot': at, 'sel': sel,
            'counts': np.array([len(crops[j]) for j in kept])}


def build_train_batch(kind, frames, frame_offsets, poses, tracks, seed, epoch, gt_boxes=None, matched=None, iou=None, enlarge=1.1,
                      bev=False, crop=True, augment_single=True):
    """every track of a batch (tracks: dict of numpy arrays with the TrackBatch fields); GRM: gt_boxes (B, L, 7), matched (B, L);
    CRM: iou (B, L).  Returns the list of per-track dicts."""
    out = []
    for b in range(len(tracks['box_num'])):
        L = int(tracks['box_num'][b])
        bx, sc = np.asarray(tracks['boxes'][b], np.float64), np.asarray(tracks['scores'][b])
        crops = track_crops(frames, frame_offsets, poses, bx, tracks['frame_of_box'][b], L, enlarge, bev, crop)
        uid = int(tracks['track_uid'][b])
        if kind == 'grm':
            out.append(geometry_train_track(crops, bx, sc, gt_boxes[b], matched[b], L, uid, seed, epoch, augment_single=augment_single))
        else:
            out.append(confidence_train_track(crops, bx, sc, iou[b], L, uid, seed, epoch))
    return out

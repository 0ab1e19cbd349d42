"""Float64 numpy restatement of the PRM training samples (detzero_b200/csrc/refine_data.cu dz_refine_train_draw kind 0 /
dz_position_train_inputs, detzero_b200/refine/data.py position_training_inputs): the training branch of
WaymoPositionDataset.extract_track_feature (refining/detzero_refine/datasets/waymo/waymo_position_dataset.py:31-184) with
AUGMENT_FULL off.  It reuses the restatements of oracle/refine_data_ref.py (crop, keyed sampler, p2co encoding, init-box frame) and
oracle/refine_train_data_ref.py (the keyed draws), and keeps their deviations: keyed draws and point samples on
(epoch_seed(seed, epoch), track_uid), float64 geometry, and the kept boxes in ascending slot order.

The PRM's draws are the CRM's rule (train_draw 'crm': kept count, kept subset, init position) over the matched slots, as the GRM's
eligible set is: random.randint(min(5, m), m), random.sample(range(m), n), np.random.randint(0, n).
"""
import numpy as np

from oracle.refine_data_ref import PRM_M, PRM_Q, _pad, encode_p2co, limit_heading, sample_ranks, track_crops
from oracle.refine_train_data_ref import init_frame_at, train_draw


def to_init_frame(init, R, boxes):
    """init_coords_transform's traj_gt: boxes (n, 7) f64 world -> the init box's frame, heading limited before and after"""
    out = np.array(boxes, np.float64)
    out[:, :3] = (out[:, :3] - init[:3]) @ R.T
    out[:, 6] = [limit_heading(limit_heading(h) - init[6]) for h in np.asarray(boxes, np.float64)[:, 6]]
    return out


def position_train_track(crops, boxes, scores, gt_boxes, matched, L, uid, seed, epoch, Lmax=200, kq=256, km=48):
    """WaymoPositionDataset.extract_track_feature (training, AUGMENT_FULL off) for one track; crops = track_crops(...)"""
    d = train_draw('crm', np.nonzero(np.asarray(matched[:L]) != 0)[0], uid, seed, epoch)
    es, kept, at = d['seed'], d['kept'], d['init']
    n = len(kept)
    bx, sc, gt = boxes[kept], np.asarray(scores)[kept], np.asarray(gt_boxes, np.float64)[kept]
    init, R, traj = init_frame_at(bx, n, at)
    q, m = np.zeros((Lmax, kq, 32)), np.zeros((Lmax, km, 32))
    sel_q, sel_m = [], []
    for i, j in enumerate(kept):
        local = crops[j].copy()
        local[:, :3] = (local[:, :3] + (bx[i, :3] - init[:3])) @ R.T
        sq = sample_ranks(len(local), kq, es, uid, i, PRM_Q)
        sm = sample_ranks(len(local), km, es, uid, i, PRM_M)
        sel_q.append(sq)
        sel_m.append(sm)
        q[i] = encode_p2co(_pad(local[sq], kq), traj[i], sc[i], None)
        m[i] = encode_p2co(_pad(local[sm], km), traj[i], sc[i], None)
    tr, gtr = np.zeros((Lmax, 7)), np.zeros((Lmax, 7))
    tr[:n], gtr[:n] = traj, to_init_frame(init, R, gt)
    mask = np.ones(Lmax)
    mask[:n] = 0
    return {'pos_query_points': q, 'pos_memory_points': m, 'pos_trajectory': tr, 'gt_pos_trajectory': gtr, 'padding_mask': mask,
            'pos_init_box': init, 'box_num': n, 'kept': kept, 'init_slot': at, 'sel': (sel_q, sel_m),
            'counts': np.array([len(crops[j]) for j in kept])}


def build_position_train_batch(frames, frame_offsets, poses, tracks, seed, epoch, gt_boxes, matched, enlarge=1.1, bev=False,
                               crop=True):
    """every track of a batch (tracks: dict of numpy arrays with the TrackBatch fields; gt_boxes (B, L, 7), matched (B, L)).
    Returns the list of per-track dicts."""
    out = []
    for b in range(len(tracks['box_num'])):
        L = int(tracks['box_num'][b])
        bx, sc = np.asarray(tracks['boxes'][b], np.float64), np.asarray(tracks['scores'][b])
        crops = track_crops(frames, frame_offsets, poses, bx, tracks['frame_of_box'][b], L, enlarge, bev, crop)
        out.append(position_train_track(crops, bx, sc, gt_boxes[b], matched[b], L, int(tracks['track_uid'][b]), seed, epoch,
                                        Lmax=len(bx)))
    return out

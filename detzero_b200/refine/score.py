"""The refiners against ground truth on the device (csrc/refine_gt.cu): the recall records of DetZero's three refine models and
the CRM's IoU labels, from the targets refine.data.track_targets attaches to a TrackBatch.

Replaces generate_recall_record of refining/detzero_refine/models/position_refine_model.py:50-169, geometry_refine_model.py:45-178
(the branch without CENTER_ALIGN) and confidence_refine_model.py:35-108, generate_refine_boxes_iou of daemon/generate_iou_gt.py:14-59,
and the ratios refining/tools/eval_utils.py:194-238 derives from the accumulated records.  The reference scores track by track on
the host (two n x n boxes_iou3d_gpu matrices per track for their diagonals, one .item() per threshold per track); here one launch
scores every track of the call, and each record is built on the host from one device-to-host copy of the per-track counts, with no
per-track read.

The records reproduce the reference's arithmetic as written, including what looks accidental:
  * the track-level ratios (boxes over the threshold / matched boxes of the track) use the first threshold of the list only;
  * the per-state track-level keys count ``ratio >= 0.7`` (PRM) or ``ratio > 0.7`` (GRM) under every threshold key, whatever the
    threshold; the keys without a state count ``ratio > threshold``;
  * the ratios pass through float32 (torch.Tensor(list)) before they are compared, and the thresholds are compared as float32;
  * the CRM record counts every box of every track, matched or not, in 'Box num', and leaves its threshold keys at 0.
Values are Python ints (the reference leaves 0-dim tensors and numpy integers in some entries).  Where the reference divides by zero (a
matched track none of whose boxes has ground truth) the track's ratios are 0.

One deliberate deviation: each pair of boxes is re-centred on its ground-truth centre in float64 before the float32 clip (see
csrc/refine_gt.cu); the reference rounds world or init-frame boxes to float32 first.

Out of scope: gt_geo_query_boxes and everything else only training reads, the losses, refiner test-time augmentation (the
reference's merge step raises NotImplementedError), CENTER_ALIGN (its branch cannot run in the reference; rejected here), the
detector's generate_recall_record, and Waymo AP / MOTA.
"""
import numpy as np
import torch

from .. import ops
from .._lib import check, darr, lib

#: POST_PROCESSING.RECALL_THRESH_LIST of the shipped refine model configs, per class
RECALL_THRESH_LIST = {'Vehicle': [0.7], 'Pedestrian': [0.5], 'Cyclist': [0.5]}
MAX_THRESHOLDS = 8
_STATES = ('static', 'dynamic')


def boxes_iou3d_aligned(boxes_a, boxes_b):
    """(N, >=7), (N, >=7) CUDA float32 rows (any row stride) -> (N) the 3-D IoU of row i with row i: the diagonal of
    track.IoU3D_dis_mat(boxes_a, boxes_b), bit for bit (iou3d_nms_utils.boxes_iou3d_gpu(a, b).diag())"""
    for t in (boxes_a, boxes_b):
        assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.shape[1] >= 7 and t.stride(1) == 1, (t.shape, t.dtype)
    n = boxes_a.shape[0]
    assert boxes_b.shape[0] == n, (boxes_a.shape, boxes_b.shape)
    out = torch.empty((n,), dtype=torch.float32, device=boxes_a.device)
    if n:
        check(lib().dz_boxes_iou3d_aligned(ops._p(boxes_a), boxes_a.stride(0), ops._p(boxes_b), boxes_b.stride(0), n, ops._p(out),
                                           ops._stream()), 'boxes_iou3d_aligned')
        ops._count(1)
    return out


def _thresholds(thresholds):
    th = [float(t) for t in thresholds]
    if not 1 <= len(th) <= MAX_THRESHOLDS:
        raise ValueError('1..%d recall thresholds (got %d)' % (MAX_THRESHOLDS, len(th)))
    return th


def score_boxes(in_boxes, out_boxes, size, tracks, targets, thresholds=()):
    """One dz_refine_score launch over the B tracks: in_boxes / out_boxes (B, L, 7) world boxes before / after refinement
    (out_boxes None: label mode, every valid slot scored), size (B, 7) or None (the refined box's dx, dy, dz).
    -> iou_in (B, L) f32, iou_out (B, L) f32 or None, rec (B, 1 + 2 T) int32 [scored slots, count(iou_in > th).., count(iou_out >
    th)..].  Device tensors, enqueue only."""
    dev = tracks.boxes.device
    B, L, th = len(tracks), tracks.L, [float(t) for t in thresholds]
    f64 = lambda t: t.to(device=dev, dtype=torch.float64).contiguous()
    in_boxes = f64(in_boxes)
    assert in_boxes.shape == (B, L, 7) and len(targets) == B, (in_boxes.shape, B, L)
    if out_boxes is not None:
        out_boxes = f64(out_boxes)
        assert out_boxes.shape == (B, L, 7), out_boxes.shape
    if size is not None:
        size = size.to(device=dev, dtype=torch.float32).reshape(B, 7).contiguous()
    iou_in = torch.zeros((B, L), dtype=torch.float32, device=dev)
    iou_out = torch.zeros((B, L), dtype=torch.float32, device=dev) if out_boxes is not None else None
    rec = torch.zeros((B, 1 + 2 * len(th)), dtype=torch.int32, device=dev)
    if B:
        check(lib().dz_refine_score(ops._p(in_boxes), ops._p(out_boxes), ops._p(size), ops._p(targets.gt_boxes.contiguous()),
                                    ops._p(targets.matched.contiguous()), ops._p(targets.matched_tracklet.contiguous()),
                                    ops._p(tracks.box_num), B, L, darr(th), len(th), ops._p(iou_in), ops._p(iou_out), ops._p(rec),
                                    ops._stream()), 'refine_score')
        ops._count(1)
    return iou_in, iou_out, rec


def empty_record(thresholds, confidence=False):
    """a record with every key of the reference's, in its order, all zero"""
    rec = {'Box num': 0, 'Track num': 0, 'static': 0, 'dynamic': 0}
    if confidence:
        rec.update({'matched_up': 0, 'matched_down': 0, 'unmatched_up': 0, 'unmatched_down': 0, 'gt_score': [], 'pred_score': [],
                    'ori_score': []})
    for th in thresholds:
        for level in ('Box', 'Track'):
            for state in ('', ' (static)', ' (dynamic)'):
                for side in ('input', 'output'):
                    rec['%s level %s%s %s' % (level, side, state, str(th))] = 0
    return rec


def record_from_counts(counts, state, matched_tracklet, thresholds, state_cut_inclusive):
    """The PRM / GRM record from the per-track host arrays: counts (B, 1 + 2 T) [matched boxes, inputs over th.., outputs over
    th..], state (B) (1 dynamic), matched_tracklet (B).  state_cut_inclusive: the per-state track-level test is ratio >= 0.7 (PRM)
    rather than ratio > 0.7 (GRM)."""
    th = [float(t) for t in thresholds]
    T = len(th)
    rec = empty_record(thresholds)
    cut = np.float32(0.7)
    for b in np.flatnonzero(np.asarray(matched_tracklet)):
        n = int(counts[b, 0])
        st = _STATES[int(state[b] != 0)]
        rec['Box num'] += n
        rec['Track num'] += 1
        rec[st] += n
        # torch.Tensor([num / obj_len]): the ratio of the first threshold, through float32
        r_in = np.float32(int(counts[b, 1]) / n) if n else np.float32(0)
        r_out = np.float32(int(counts[b, 1 + T]) / n) if n else np.float32(0)
        for k, t in enumerate(thresholds):
            s = str(t)
            rec['Box level input %s' % s] += int(counts[b, 1 + k])
            rec['Box level output %s' % s] += int(counts[b, 1 + T + k])
            rec['Box level input (%s) %s' % (st, s)] += int(counts[b, 1 + k])
            rec['Box level output (%s) %s' % (st, s)] += int(counts[b, 1 + T + k])
            rec['Track level input %s' % s] += int(r_in > np.float32(th[k]))
            rec['Track level output %s' % s] += int(r_out > np.float32(th[k]))
            rec['Track level input (%s) %s' % (st, s)] += int(r_in >= cut if state_cut_inclusive else r_in > cut)
            rec['Track level output (%s) %s' % (st, s)] += int(r_out >= cut if state_cut_inclusive else r_out > cut)
    return rec


def _recall(in_boxes, out_boxes, size, tracks, targets, thresholds, inclusive):
    th = _thresholds(thresholds)
    _, _, rec = score_boxes(in_boxes, out_boxes, size, tracks, targets, th)
    host = torch.cat([rec, targets.state.to(torch.int32)[:, None], targets.matched_tracklet.to(torch.int32)[:, None]], 1).cpu().numpy()
    return record_from_counts(host[:, :-2], host[:, -2], host[:, -1], list(thresholds), inclusive)


def position_recall(pred_world, tracks, targets, thresholds):
    """PositionRefineModel.generate_recall_record for the B tracks of the call: the tracker's boxes (tracks.boxes) on the input side,
    pred_world (B, L, 7), revert_position_boxes' world boxes, on the output side, against targets.gt_boxes on the slots where the
    track and the box are matched.  One launch, one device-to-host copy of the per-track counts.  Returns the reference's dict
    (keys and order: 'Box num', 'Track num', 'static', 'dynamic', then per threshold 'Box level input <th>', 'Box level output
    <th>', their (static) / (dynamic) forms, and the same six 'Track level' keys); see the module docstring for the arithmetic."""
    return _recall(tracks.boxes, pred_world, None, tracks, targets, thresholds, True)


def geometry_recall(grm_pred, tracks, targets, thresholds, center_align=False):
    """GeometryRefineModel.generate_recall_record (without CENTER_ALIGN): the tracker's boxes on the input side; on the output side
    the same boxes with the size grm_pred[b][3:6] (geometry_refine_model.py:105-108), put together inside the kernel.  grm_pred
    (B, 7).  One launch, one copy; the dict as position_recall's."""
    if center_align:
        raise ValueError('CENTER_ALIGN is not supported (the reference branch indexes per_gt_traj[idx] and cannot run)')
    return _recall(tracks.boxes, tracks.boxes, grm_pred, tracks, targets, thresholds, False)


def refine_iou_labels(prm_world, grm_pred, tracks, targets):
    """generate_refine_boxes_iou: the 3-D IoU of every box (the PRM world box prm_world (B, L, 7) with the GRM size grm_pred[b][3:6])
    with its ground-truth box -> (B, L) float32 on the device: 0 where there is no ground truth (the reference's zero box), matched
    track or not, and -1 past box_num (the padding WaymoConfidenceDataset applies).  Enqueue only."""
    iou, _, _ = score_boxes(prm_world, None, grm_pred, tracks, targets)
    pad = torch.arange(tracks.L, device=iou.device)[None, :] >= tracks.box_num[:, None]
    return iou.masked_fill_(pad, -1.0)


def confidence_recall(conf_score, pred_score, iou, tracks, targets, thresholds):
    """ConfidenceRefineModel.generate_recall_record: conf_score (the tracker's per-box scores, confidence_inputs' 'conf_score'),
    pred_score (the CRM's) and iou (refine_iou_labels), each (B, L).  The four counters per track come from one launch
    (dz_confidence_score); they and the per-box scores of the 'gt_score' / 'pred_score' / 'ori_score' lists reach the host in one
    copy."""
    th = _thresholds(thresholds)
    dev = tracks.boxes.device
    B, L = len(tracks), tracks.L
    f32 = lambda t: t.to(device=dev, dtype=torch.float32).reshape(B, L).contiguous()
    conf, pred, iou = f32(conf_score), f32(pred_score), f32(iou)
    cnt = torch.zeros((B, 5), dtype=torch.int32, device=dev)
    if B:
        check(lib().dz_confidence_score(ops._p(conf), ops._p(pred), ops._p(iou), ops._p(tracks.box_num), B, L, ops._p(cnt),
                                        ops._stream()), 'confidence_score')
        ops._count(1)
    ints = torch.cat([cnt, targets.matched_tracklet.to(torch.int32)[:, None]], 1)
    # one copy: the integer records travel as their float32 bit patterns beside the scores
    host = torch.cat([ints.reshape(-1).view(torch.float32), conf.reshape(-1), pred.reshape(-1), iou.reshape(-1)]).cpu().numpy()
    ints = host[:B * 6].view(np.int32).reshape(B, 6)
    conf, pred, iou = (host[B * 6 + k * B * L:B * 6 + (k + 1) * B * L].reshape(B, L) for k in range(3))
    rec = empty_record(thresholds, confidence=True)
    for b in range(B):
        n = int(ints[b, 4])
        rec['ori_score'].extend(conf[b, :n])
        rec['pred_score'].extend(pred[b, :n])
        rec['gt_score'].extend(iou[b, :n] >= np.float32(0.7))
        for k, key in enumerate(('matched_up', 'matched_down', 'unmatched_up', 'unmatched_down', 'Box num')):
            rec[key] += int(ints[b, k])
    rec['Track num'] += int(ints[:, 5].sum())
    return rec


def accumulate(a, b):
    """the sum of two records of the same thresholds, as eval_one_epoch adds them up batch after batch (counts add, the CRM's lists
    extend); an empty dict is the neutral element"""
    if not a or not b:
        return {k: (list(v) if isinstance(v, list) else v) for k, v in (a or b).items()}
    if list(a) != list(b):
        raise ValueError('records of different thresholds or models')
    return {k: (list(a[k]) + list(b[k]) if isinstance(a[k], list) else a[k] + b[k]) for k in a}


def summarize(record, thresholds):
    """The ratios eval_one_epoch returns (refining/tools/eval_utils.py:194-238): per threshold 'Recall@box/input_<th>',
    'Recall@box/output_<th>' (over max(Box num, 1)), 'Recall@track/input_<th>', 'Recall@track/output_<th>' (over max(Track num,
    1))"""
    out = {}
    nb, nt = max(record['Box num'], 1), max(record['Track num'], 1)
    for th in thresholds:
        s = str(th)
        out['Recall@box/input_%s' % s] = record['Box level input %s' % s] / nb
        out['Recall@box/output_%s' % s] = record['Box level output %s' % s] / nb
        out['Recall@track/input_%s' % s] = record['Track level input %s' % s] / nt
        out['Recall@track/output_%s' % s] = record['Track level output %s' % s] / nt
    return out

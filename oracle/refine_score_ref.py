"""numpy restatement (float64) of how DetZero scores its refiners against ground truth: the per-track targets of
daemon/prepare_object_data.py:64-190, the gt_pos_trajectory of waymo_position_dataset.py:76-80 (init_coords_transform), the recall
records of PositionRefineModel / GeometryRefineModel / ConfidenceRefineModel.generate_recall_record
(refining/detzero_refine/models/*_refine_model.py) and the CRM's IoU labels (daemon/generate_iou_gt.py:14-59).

Inputs are the reference's pickle-shaped dicts: ``attach_targets`` takes what target_assign.assign_track_target returns for one
sequence ({'label': {id: {'track', 'gt'}}, 'unlabel': {id: {'track'}}}, e.g. oracle.track_gt_ref.assign_track_target) and returns
the per-object infos the refining datasets read ({id: {'boxes_global', 'gt_boxes_global', 'matched', 'matched_tracklet', 'state',
'name', 'score', 'sample_idx'}}).

The rotated clip is the oracle's C restatement (float32, as the reference's op).  With ``centre=True`` (the device's arithmetic,
csrc/refine_gt.cu) each pair of boxes is moved to its ground-truth centre in float64 before it is rounded to float32; with
``centre=False`` the boxes are rounded where they stand, as the reference does.  Ratios and thresholds are compared in float32, as
torch compares them there.

Every record function also returns its decision ``margin``: the smallest |iou - threshold| over the scored boxes ('iou'; for the
CRM |iou - 0.7| and |pred - ori|), and the smallest |ratio - cut| over the track-level ratios ('ratio').  A device result may
differ from the oracle's only where a margin is small.
"""
import numpy as np

from . import boxes_iou3d
from .track_ref import Margin

PI = np.pi


def limit_heading_range(a):
    a = np.array(a, np.float64, copy=True)
    for _ in range(8):
        a = np.where(a >= PI, a - 2 * PI, a)
        a = np.where(a < -PI, a + 2 * PI, a)
    return a


def attach_targets(assigned, class_name=None):
    """prepare_object_data.py:64-190, regrouped per object as its step 2 does -> {track id: info}, labelled tracks first"""
    out = {}
    for tid, lab in assigned['label'].items():
        t, g = lab['track'], lab['gt']
        if class_name is not None and class_name not in t['name']:
            continue
        boxes = np.asarray(t['boxes_global'], np.float64)[:, :7]
        gtb = np.zeros_like(boxes)
        matched = np.zeros(len(boxes), bool)
        gsid = np.asarray(g['sample_idx']).astype(str)
        for j, sid in enumerate(np.asarray(t['sample_idx']).astype(str)):
            hit = np.flatnonzero(gsid == sid)
            if len(hit):
                gtb[j] = np.asarray(g['gt_boxes_global'], np.float64)[hit[0], :7]
                matched[j] = True
        out[tid] = {'boxes_global': boxes, 'gt_boxes_global': gtb, 'matched': matched, 'matched_tracklet': True,
                    'state': t['state'], 'name': str(t['name'][0]), 'score': np.asarray(t['score'], np.float32),
                    'sample_idx': np.asarray(t['sample_idx'])}
    for tid, lab in assigned['unlabel'].items():
        t = lab['track']
        if class_name is not None and class_name not in t['name']:
            continue
        boxes = np.asarray(t['boxes_global'], np.float64)[:, :7]
        out[tid] = {'boxes_global': boxes, 'gt_boxes_global': np.zeros_like(boxes), 'matched': np.ones(len(boxes), bool),
                    'matched_tracklet': False, 'state': t['state'], 'name': str(t['name'][0]),
                    'score': np.asarray(t['score'], np.float32), 'sample_idx': np.asarray(t['sample_idx'])}
    return out


def init_frame_boxes(boxes, init_box):
    """init_coords_transform on a trajectory: world boxes (n, 7) in the frame of init_box, float64"""
    b = np.array(boxes, np.float64, copy=True)[:, :7]
    yaw = limit_heading_range(init_box[6])
    c, s = np.cos(yaw), np.sin(yaw)
    d = b[:, :3] - np.asarray(init_box, np.float64)[:3]
    b[:, 0], b[:, 1], b[:, 2] = c * d[:, 0] + s * d[:, 1], -s * d[:, 0] + c * d[:, 1], d[:, 2]
    b[:, 6] = limit_heading_range(limit_heading_range(b[:, 6]) - yaw)
    return b


def world_boxes(pred, init_box):
    """box_coords_transform (revert_to_each_frame): boxes in the frame of init_box back to the world, float64"""
    p = np.asarray(pred, np.float64)[:, :7]
    yaw = limit_heading_range(init_box[6])
    c, s = np.cos(yaw), np.sin(yaw)
    w = p.copy()
    w[:, 0], w[:, 1], w[:, 2] = c * p[:, 0] - s * p[:, 1] + init_box[0], s * p[:, 0] + c * p[:, 1] + init_box[1], p[:, 2] + init_box[2]
    w[:, 6] = limit_heading_range(p[:, 6] + yaw)
    return w


def gt_pos_trajectory(info):
    """the dataset's gt_pos_trajectory (eval): gt_boxes_global in the frame of the track's middle box"""
    return init_frame_boxes(info['gt_boxes_global'], info['boxes_global'][len(info['boxes_global']) // 2])


def aligned_iou(boxes, gt, centre=True):
    """3-D IoU of boxes[i] with gt[i] -> (n) float32"""
    a, g = np.array(boxes, np.float64)[:, :7], np.array(gt, np.float64)[:, :7]
    if centre:
        a[:, :3] -= g[:, :3]
        g[:, :3] = 0
    out = np.zeros(len(a), np.float32)
    for i in range(len(a)):
        if g[i, 3] * g[i, 4] * g[i, 5] > 0:
            out[i] = boxes_iou3d(a[i:i + 1].astype(np.float32), g[i:i + 1].astype(np.float32))[0, 0]
    return out


def empty_record(thresholds, confidence=False):
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


def box_recall(infos, out_boxes, thresholds, inclusive, centre=True):
    """The PRM (inclusive=True) / GRM (False) record over the tracks ``infos`` (dict order), out_boxes[i] (n_i, 7) the world boxes
    after refinement -> (record, per-track (iou_in, iou_out) over the matched boxes, margin)"""
    rec, margin, ious = empty_record(thresholds), {'iou': Margin(), 'ratio': Margin()}, []
    cut = np.float32(0.7)
    for info, ob in zip(infos.values(), out_boxes):
        if not info['matched_tracklet']:
            ious.append(None)
            continue
        m = info['matched']
        i_in = aligned_iou(info['boxes_global'][m], info['gt_boxes_global'][m], centre)
        i_out = aligned_iou(np.asarray(ob)[m], info['gt_boxes_global'][m], centre)
        ious.append((i_in, i_out))
        n, st = int(m.sum()), info['state']
        rec['Box num'] += n
        rec['Track num'] += 1
        rec[st] += n
        t0 = np.float32(thresholds[0])
        r_in = np.float32(int((i_in > t0).sum()) / n) if n else np.float32(0)
        r_out = np.float32(int((i_out > t0).sum()) / n) if n else np.float32(0)
        margin['ratio'].add([r_in, r_out], float(cut), 'ratio vs 0.7')
        for th in thresholds:
            s, t32 = str(th), np.float32(th)
            margin['iou'].add(np.concatenate([i_in, i_out]), float(t32), 'iou vs %s' % s)
            margin['ratio'].add([r_in, r_out], float(t32), 'ratio vs %s' % s)
            for side, v, r in (('input', i_in, r_in), ('output', i_out, r_out)):
                k = int((v > t32).sum())
                rec['Box level %s %s' % (side, s)] += k
                rec['Box level %s (%s) %s' % (side, st, s)] += k
                rec['Track level %s %s' % (side, s)] += int(r > t32)
                rec['Track level %s (%s) %s' % (side, st, s)] += int(r >= cut if inclusive else r > cut)
    return rec, ious, margin


def position_recall(infos, pred_world, thresholds, centre=True):
    return box_recall(infos, pred_world, thresholds, True, centre)


def geometry_out_boxes(infos, grm_pred):
    """geometry_refine_model.py:105-108: the track's boxes with the predicted size"""
    out = []
    for info, p in zip(infos.values(), grm_pred):
        b = info['boxes_global'].copy()
        b[:, 3:6] = np.asarray(p, np.float32)[3:6]
        out.append(b)
    return out


def geometry_recall(infos, grm_pred, thresholds, centre=True):
    return box_recall(infos, geometry_out_boxes(infos, grm_pred), thresholds, False, centre)


def refine_iou_labels(infos, prm_world, grm_pred, centre=True):
    """generate_refine_boxes_iou: per track the IoU of (PRM box, GRM size) with the ground-truth box, every box"""
    out = []
    for info, pw, p in zip(infos.values(), prm_world, grm_pred):
        b = np.array(pw, np.float64)[:, :7]
        b[:, 3:6] = np.asarray(p, np.float32)[3:6]
        out.append(aligned_iou(b, info['gt_boxes_global'], centre))
    return out


def confidence_recall(infos, conf_score, pred_score, iou, thresholds):
    """ConfidenceRefineModel.generate_recall_record; conf_score / pred_score / iou: per track (n_i) float32 -> (record, margin)"""
    rec, margin = empty_record(thresholds, confidence=True), {'iou': Margin(), 'score': Margin()}
    for info, ori, pred, gt in zip(infos.values(), conf_score, pred_score, iou):
        ori, pred, gt = np.asarray(ori, np.float32), np.asarray(pred, np.float32), np.asarray(gt, np.float32)
        lab = gt >= np.float32(0.7)
        margin['iou'].add(gt, float(np.float32(0.7)), 'iou vs 0.7')
        margin['score'].add(pred, ori, 'pred vs ori')
        rec['ori_score'].extend(ori)
        rec['pred_score'].extend(pred)
        rec['gt_score'].extend(lab)
        mu, md, uu = int((lab & (pred >= ori)).sum()), int((lab & (pred < ori)).sum()), int(((gt < np.float32(0.7)) & (pred >= ori)).sum())
        rec['matched_up'] += mu
        rec['matched_down'] += md
        rec['unmatched_up'] += uu
        rec['unmatched_down'] += len(ori) - mu - md - uu
        rec['Box num'] += len(ori)
        rec['Track num'] += int(bool(info['matched_tracklet']))
    return rec, margin

"""The DetZero refiner stage over a whole tracked sequence, and the combine stage after it (daemon/combine_output.py), on the device:
from the tracker's result and the sequence's points to the per-frame result the reference evaluator reads.

``refine_sequence`` runs, for each class, the PRM, GRM and (optionally) CRM inputs and models chunk by chunk over the class's tracks,
reverts the PRM boxes to each frame, and combines every class in one ``refine.data.combine_frames`` call (csrc/combine.cu).
"""
import numpy as np
import torch

from .refine import data as rdata
from .refine import score as rscore
from .track import CLASS_NAMES


class OffboardResult:
    """Final boxes of one sequence: rows (F, R, 9) f32 [x, y, z, dx, dy, dz, heading, score, label], obj_id (F, R) int32 (-1: a
    dropped detection), count (F) int32 (see refine.data.combine_frames), and the per-track tables they came from, in output order:
    tables['prm_lidar'] (B, L, 7) f64, 'grm_pred' (B, 7) f32, 'scores' (B, L) f32, 'frame_of_box' (B, L), 'box_num' (B), 'cls' (B),
    'track_id' (B) int64; poses (F, 4, 4) f64.  When the sequence was scored against ground truth (refine_sequence(assign=...)):
    recall {class: {'PRM', 'GRM', 'CRM': the refine.score record}} and tables['refine_iou'] (B, L) f32 (the CRM's IoU labels, -1
    past box_num), tables['matched'] (B, L) uint8; recall is None otherwise."""

    def __init__(self, tables, poses, rows, obj_id, count, recall=None):
        self.tables, self.poses, self.rows, self.obj_id, self.count = tables, poses, rows, obj_id, count
        self.recall = recall

    def frame_order(self):
        """the sequence frame indices that have rows, in order of first appearance over the tracks (convert_frame_format's order)"""
        fob = self.tables['frame_of_box'].cpu().numpy()
        bn = self.tables['box_num'].cpu().numpy()
        seen = fob[np.arange(fob.shape[1])[None, :] < bn[:, None]]
        _, first = np.unique(seen, return_index=True)
        return seen[np.sort(first)]

    def to_reference(self, sequence_name, frame_ids):
        """The frame list combine_final pickles as <class>_final_frame.pkl, for this sequence: one dict per frame with 'sequence_name',
        'frame_id' (int(frame_ids[f])), 'obj_ids' (int64, the track rows only), 'name' (object), 'score', 'boxes_lidar' (float32),
        'boxes_global' (zeros, one row per track row, as convert_frame_format leaves it when boxes_lidar is present) and 'pose', in
        order of first appearance over the tracks (not sorted)."""
        rows, oid, cnt = self.rows.cpu().numpy(), self.obj_id.cpu().numpy(), self.count.cpu().numpy()
        poses = self.poses.cpu().numpy()
        out = []
        for f in self.frame_order():
            n = int(cnt[f])
            r, ids = rows[f, :n], oid[f, :n]
            t = int((ids >= 0).sum())
            out.append({'sequence_name': sequence_name, 'frame_id': int(frame_ids[f]), 'obj_ids': ids[:t].astype(np.int64),
                        'name': np.array([CLASS_NAMES[int(c) - 1] for c in r[:, 8]], dtype=object), 'score': r[:, 7].copy(),
                        'boxes_lidar': r[:, :7].copy(), 'boxes_global': np.zeros((t, 9), np.float32), 'pose': poses[f].copy()})
        return out


def _forward(model, inputs, key):
    out = model(dict(inputs))
    return out[0][key] if isinstance(out, tuple) else out['pred_score' if key == 'pred_score' else 'batch_box_preds']


class _Stages:
    """device time per stage from CUDA events, read once at the end"""

    def __init__(self, timings):
        self.timings, self.events = timings, []

    def mark(self, name):
        if self.timings is None:
            return
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.events.append((name, e))

    def finish(self):
        if self.timings is None or not self.events:
            return
        self.events[-1][1].synchronize()
        for (name, a), (_, b) in zip(self.events, self.events[1:]):
            if name is not None:
                self.timings[name] = self.timings.get(name, 0.0) + a.elapsed_time(b)


def refine_sequence(frames, frame_offsets, poses, track_result, models, sequence=0, class_names=CLASS_NAMES, combine_conf_res=True,
                    combine_drop=True, chunk=16, seed=0, max_rows=1024, timings=None, assign=None, recall_thresholds=None):
    """DetZero's refine and combine stages over one tracked sequence (refining/tools/test.py per class, then combine_final).
    frames / frame_offsets / poses: the sequence's collated points, as refine.data.position_inputs takes them (frame f of the tracker
    is frame f here).  track_result: track.TrackResult, sequence ``sequence`` of it.  models: {class name: {'PRM', 'GRM', 'CRM':
    refine.RefineTemplate (or the bare module)}}; PRM and GRM are required for every listed class, CRM only with combine_conf_res.
    For each class in class_names order: its tracks (track_batch, ids ascending), in chunks of ``chunk`` tracks, the PRM, GRM and
    CRM inputs (keyed by ``seed``) and forwards, and revert_position_boxes.  Then one refine.data.combine_frames over every class:
    the PRM box with the GRM size, the CRM score (the tracker's per-box score when combine_conf_res is False), and, with
    combine_drop, the tracker's dropped detections of every class.  Tracks of unlisted classes are left out.
    timings: an optional dict that receives the device milliseconds of each stage (inputs, forwards, revert, combine; one extra
    synchronisation).  Returns an OffboardResult.
    assign: a track.AssignResult of ``track_result`` (track.assign_track_target); each chunk then also gets its ground truth
    (refine.data.track_targets, stage 'targets') and is scored (refine.score: the PRM, GRM and, with combine_conf_res, CRM records
    and the IoU labels, stage 'score'; one device-to-host copy per record and chunk), and the chunks' records are added up per
    class into OffboardResult.recall.  recall_thresholds: {class: list}, by default refine.score.RECALL_THRESH_LIST.  Without
    ``assign`` none of this runs.
    Deviations from combine_final: the reference writes one file per class and its class loop accumulates, so each file holds every
    class processed so far, and its last file omits sequences without a track of the last class; here one call gives all listed
    classes of its sequence.  combine_det raises KeyError for a frame with tracks but no drop entry; here that frame has no
    dropped row."""
    for c in class_names:
        if c not in CLASS_NAMES:
            raise ValueError('unknown class %r' % (c,))
        need = ('PRM', 'GRM', 'CRM') if combine_conf_res else ('PRM', 'GRM')
        missing = [k for k in need if k not in models.get(c, {})]
        if missing:
            raise KeyError('models[%r] lacks %s' % (c, ', '.join(missing)))
    thresholds = dict(rscore.RECALL_THRESH_LIST)
    thresholds.update(recall_thresholds or {})
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError('chunk must be positive')
    dev = track_result.trk.device
    F = len(frame_offsets) - 1
    if F != int(track_result.num_frames[sequence]):
        raise ValueError('%d frames given for a sequence the tracker ran over %d frames' % (F, int(track_result.num_frames[sequence])))
    poses = torch.as_tensor(poses).to(device=dev, dtype=torch.float64).contiguous()
    st = _Stages(timings)
    parts = {k: [] for k in ('prm_lidar', 'grm_pred', 'scores', 'frame_of_box', 'box_num', 'cls', 'track_id')}
    recall = None
    if assign is not None:
        parts['refine_iou'], parts['matched'] = [], []
        recall = {c: {k: rscore.empty_record(thresholds[c], k == 'CRM') for k in (('PRM', 'GRM', 'CRM') if combine_conf_res
                                                                                  else ('PRM', 'GRM'))} for c in class_names}
    for c in class_names:
        tb = track_result.track_batch(c, sequence=sequence)
        m = models[c]
        for c0 in range(0, len(tb), chunk):
            sub = tb.select(slice(c0, c0 + chunk))
            if assign is not None:
                st.mark('targets')
                tg = rdata.track_targets(assign, sub, sequence)
            st.mark('position_inputs')
            pin = rdata.position_inputs(frames, frame_offsets, poses, sub, seed=seed)
            st.mark('prm_forward')
            pred = _forward(m['PRM'], pin, 'pred_boxes')
            st.mark('geometry_inputs')
            gin = rdata.geometry_inputs(frames, frame_offsets, poses, sub, seed=seed)
            st.mark('grm_forward')
            size = _forward(m['GRM'], gin, 'pred_boxes')
            if combine_conf_res:
                st.mark('confidence_inputs')
                cin = rdata.confidence_inputs(frames, frame_offsets, poses, sub, seed=seed)
                st.mark('crm_forward')
                score = _forward(m['CRM'], cin, 'pred_score')
            else:
                score = sub.scores
            st.mark('revert')
            lidar, world = rdata.revert_position_boxes(pred, poses, sub)
            if assign is not None:
                st.mark('score')
                th, size7 = thresholds[c], size.float().reshape(len(sub), 7)
                iou = rscore.refine_iou_labels(world, size7, sub, tg)
                new = {'PRM': rscore.position_recall(world, sub, tg, th), 'GRM': rscore.geometry_recall(size7, sub, tg, th)}
                if combine_conf_res:
                    new['CRM'] = rscore.confidence_recall(sub.scores, score, iou, sub, tg, th)
                for k, r in new.items():
                    recall[c][k] = rscore.accumulate(recall[c][k], r)
                parts['refine_iou'].append(iou)
                parts['matched'].append(tg.matched)
            st.mark(None)
            parts['prm_lidar'].append(lidar)
            parts['grm_pred'].append(size.float().reshape(len(sub), 7))
            parts['scores'].append(score.float().reshape(len(sub), sub.L))
            parts['frame_of_box'].append(sub.frame_of_box)
            parts['box_num'].append(sub.box_num)
            parts['cls'].append(sub.cls)
            parts['track_id'].append(sub.track_uid)
    L = 200 if not parts['prm_lidar'] else parts['prm_lidar'][0].shape[1]
    empty = {'prm_lidar': (0, L, 7), 'grm_pred': (0, 7), 'scores': (0, L), 'frame_of_box': (0, L), 'box_num': (0,), 'cls': (0,),
             'track_id': (0,), 'refine_iou': (0, L), 'matched': (0, L)}
    dtypes = {'prm_lidar': torch.float64, 'grm_pred': torch.float32, 'scores': torch.float32, 'track_id': torch.int64,
              'refine_iou': torch.float32, 'matched': torch.uint8}
    tables = {k: torch.cat(v) if v else torch.zeros(empty[k], dtype=dtypes.get(k, torch.int32), device=dev) for k, v in parts.items()}
    drop = (track_result.boxes[sequence], track_result.counts[sequence], track_result.kept[sequence]) if combine_drop else None
    st.mark('combine')
    rows, obj_id, count = rdata.combine_frames(tables['prm_lidar'], tables['grm_pred'], tables['scores'], tables['frame_of_box'],
                                               tables['box_num'], tables['cls'], tables['track_id'], F, drop=drop, max_rows=max_rows)
    st.mark(None)
    st.finish()
    return OffboardResult(tables, poses, rows, obj_id, count, recall)

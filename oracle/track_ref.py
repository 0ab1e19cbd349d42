"""numpy restatement of the DetZero tracker (tracking/tools/cfgs/tk_model_cfgs/waymo_detzero_track.yaml with
tk_dataset_cfgs/waymo_dataset.yaml): detection pre-processing (datasets/data_processor.py), forward and reverse tracking
(models/tracking_modules/track_manager.py, kalman_filter/kalman_filter.py, data_association/), post-processing (post_process.py).

The dtypes follow the reference: a track's KF state starts as float32 and becomes float64 after its first measurement update, P / Q /
K stay float32, the association boxes are float32 world boxes, the emitted boxes mix float64 detections with float32 state.  The
assignment is scipy's linear_sum_assignment on the reference's own cost construction (1 - affinity, 5000 where cost >= 1).

One deliberate deviation: a sequence whose first frames have no track entries makes the reference's reverse pass raise KeyError; here
such frames are empty, as in csrc/tracker.cu.

``margin`` is the smallest distance from a threshold over every compared value: IoU and overlap ratios against their thresholds, the
vehicle speed clamp, the 1e-4 motion test of tracks whose hit boxes all lie within the sum of half-diagonals plus 0.05 m of each other
(any pair farther apart overlaps by exactly 0 and makes the track dynamic; so does a pair of disjoint boxes, whose clipped overlap is
exactly 0 and is left out), and per association component the cost gap to the best assignment that
avoids one chosen edge.  Where it is at least 1e-3, float rounding differences cannot change a decision.
"""
import numpy as np
from scipy.optimize import linear_sum_assignment
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from . import boxes_iou_bev, boxes_overlap_bev

CLASS_NAMES = ('Vehicle', 'Pedestrian', 'Cyclist')
PI2 = np.pi * 2


def yaw_filter(yaw):
    """transform_utils.yaw_filter, ndarray branch (dtype kept)"""
    y = np.array(yaw, copy=True)
    big = np.abs(y) >= PI2
    y[big] = y[big] - np.floor(y[big] / PI2) * PI2
    y[y > np.pi] -= PI2
    y[y <= -np.pi] += PI2
    return y


def _far(a, b, slack=0.05):
    """(N, M) True where two boxes cannot touch: centre distance above the sum of half-diagonals plus slack"""
    ra = 0.5 * np.hypot(a[:, 3], a[:, 4]).astype(np.float64)
    rb = 0.5 * np.hypot(b[:, 3], b[:, 4]).astype(np.float64)
    d = np.hypot(a[:, None, 0].astype(np.float64) - b[None, :, 0], a[:, None, 1].astype(np.float64) - b[None, :, 1])
    return d > ra[:, None] + rb[None, :] + slack


def _near_matrix(fn, a, b, near):
    """fn(a, b) where near, 0 elsewhere (a far pair has exactly 0 overlap), computed one row at a time"""
    out = np.zeros((len(a), len(b)), np.float32)
    for i in np.flatnonzero(near.any(1)):
        js = np.flatnonzero(near[i])
        out[i, js] = fn(a[i:i + 1], b[js])[0]
    return out


class Margin:
    def __init__(self):
        self.value = np.inf
        self.where = None

    def add(self, values, thr, where):
        v = np.abs(np.asarray(values, np.float64) - np.asarray(thr, np.float64))
        if v.size and v.min() < self.value:
            self.value, self.where = float(v.min()), where


class _Track:
    """KalmanFilter of kalman_filter.py (x: [x, y, z, vx, vy])"""

    def __init__(self, box, cls, score, frame, tid, cfg, dt):
        self.size = np.asarray(box[3:6])
        self.heading = box[6]
        self.cls, self.score, self.frame, self.id = cls, score, frame, tid
        self.x = np.zeros((5, 1), np.float32)
        self.x[:3, 0] = box[:3]
        self.bbox = np.zeros(9, np.float32)
        self.bbox[:7] = box[:7]
        self.F = np.eye(5, dtype=np.float32)
        self.F[0, 3] = self.F[1, 4] = np.float32(dt)
        p, q = cfg['FILTER']['P'], cfg['FILTER']['Q']
        self.P = np.diag(np.array([p[0]] * 3 + [p[1]] * 2, np.float32))
        self.Q = np.diag(np.array([q[0]] * 3 + [q[1]] * 2, np.float32))
        self.R = np.eye(3, dtype=np.float32) * np.float32(cfg['FILTER']['R'])
        self.hit = 1

    def predict(self, frame, margin):
        self.frame = frame
        x = self.x.copy()
        if self.cls == 1:
            speed, lim = np.linalg.norm(x[3:]), np.max(self.size) / 2.
            margin.add(speed, lim, 'speed clamp')
            if speed <= lim:
                x[3:] = 0.
        self.x = self.F @ x
        self.P = self.F @ self.P @ self.F.T + self.Q
        self.Q = self.Q * np.float32(1.5)
        self.hit = 0
        self.bbox = np.concatenate((self.x[:3, 0], self.size, [self.heading], self.x[3:5, 0]))
        return self.bbox

    def update(self, box, cls, score, stage2):
        self.score = score
        if stage2:
            self.hit = 2
            return
        self.hit = 1
        self.cls = cls
        z = box[:3].reshape(3, 1)
        self.size, self.heading = box[3:6], box[6]
        H = np.eye(3, 5, dtype=np.float32)
        S = H @ self.P @ H.T + self.R
        K = self.P @ H.T @ np.linalg.inv(S)
        self.x = self.x + K @ (z - H @ self.x)
        self.P = self.P - K @ H @ self.P
        self.x[:3] = z
        self.bbox = np.concatenate((box[:3], self.size, [self.heading], self.x[3:5, 0]))


def _assign(aff_ok, aff, margin, where):
    """GNN_assignment on 1 - affinity: (rows, cols) matched pairs, plus the per-component cost gap in the margin"""
    N, M = aff.shape
    if N == 0 or M == 0:
        return np.zeros((0, 2), np.int64)
    cost = (np.float32(1.0) - np.where(aff_ok, aff, np.float32(0))).astype(np.float32)
    cost[cost >= 1] = 5000.
    r, c = linear_sum_assignment(cost)
    keep = cost[r, c] < 1
    pairs = np.stack([r[keep], c[keep]], 1)
    ei, ej = np.nonzero(aff_ok)
    if len(ei) > 1:
        g = coo_matrix((np.ones(len(ei)), (ei, N + ej)), shape=(N + M, N + M))
        _, lab = connected_components(g, directed=False)
        for comp in np.unique(lab[ei]):
            rows, cols = np.flatnonzero(lab[:N] == comp), np.flatnonzero(lab[N:] == comp)
            if len(rows) * len(cols) < 2:
                continue
            sub = cost[np.ix_(rows, cols)].astype(np.float64)
            rr, cc = linear_sum_assignment(sub)
            best = sub[rr, cc].sum()
            for a, b in zip(rr, cc):
                if sub[a, b] >= 1:
                    continue
                alt = sub.copy()
                alt[a, b] = 5000.
                r2, c2 = linear_sum_assignment(alt)
                margin.add(alt[r2, c2].sum() - best, 0., where + ' assignment gap')
    return pairs


def _affinity(tk_boxes, tk_cls, det_boxes, det_cls, thr, margin, where):
    """IoUBEV_dis_mat on float32 world boxes, class mask, per-track-class threshold -> (valid edge mask (T, D), affinity)"""
    a, b = np.asarray(tk_boxes, np.float32)[:, :7], np.asarray(det_boxes, np.float32)[:, :7]
    if len(a) == 0 or len(b) == 0:
        return np.zeros((len(a), len(b)), bool), np.zeros((len(a), len(b)), np.float32)
    same = tk_cls[:, None] == det_cls[None, :]
    near = same & ~_far(a, b)
    iou = _near_matrix(boxes_iou_bev, a, b, near)
    t = np.float32(np.asarray(thr)[tk_cls - 1])[:, None] * np.ones_like(iou)
    margin.add(iou[near], t[near], where)
    return same & (iou >= t), iou


def _merge(boxes, cls, ids, thr, margin):
    """overlap_track_merge: the indices of the tracks that are deprecated"""
    n = len(boxes)
    if n == 0:
        return []
    b = np.asarray(boxes, np.float32)[:, :7]
    near = (cls[:, None] == cls[None, :]) & ~_far(b, b)
    ov = _near_matrix(boxes_overlap_bev, b, b, near)
    area = b[:, 3] * b[:, 4]
    ratio = ov / (area[:, None] + np.float32(1e-9))
    tt = np.float32(np.asarray(thr)[cls - 1])[:, None] * np.ones_like(ratio)
    margin.add(ratio[near], tt[near], 'merge ratio')
    fresh = np.ones(n, bool)
    dep = []
    for i in range(n):
        if not fresh[i]:
            continue
        s = np.flatnonzero(fresh & (ratio[i] >= tt[i]))
        best = s[np.argmin(ids[s])]
        fresh[s] = False
        dep += [j for j in s if j != best]
    return sorted(dep)


def preprocess(boxes, count, pose, cfg, margin):
    """heading_process, overlap_box_filter (max_score), transform_to_global for one frame.
    -> lidar boxes (n, 7) f32 after the heading filter, score, class, kept mask, world boxes (n, 7) f64"""
    d = np.asarray(boxes[:count], np.float32)
    lid = d[:, :7].copy()
    lid[:, 6] = yaw_filter(lid[:, 6])
    score, cls = d[:, 7].copy(), d[:, 8].astype(np.int64)
    n = len(d)
    kept = np.zeros(n, bool)
    if n:
        near = ~_far(lid, lid)
        ratio = _near_matrix(boxes_overlap_bev, lid, lid, near) / (lid[:, 3] * lid[:, 4])[:, None]
        t = np.float32(np.asarray(cfg['OVERLAP_FILTER']['CLASS_THRESHOLD'])[cls - 1])
        margin.add(ratio[near], (t[:, None] * np.ones_like(ratio))[near], 'overlap filter')
        for i in range(n):
            if kept[i]:
                continue
            s = np.flatnonzero(ratio[i] >= t[i])
            kept[s[np.argsort(score[s], kind='stable')[-1]]] = True
    c = np.concatenate([lid[:, :3], np.ones((n, 1))], 1) @ pose.T
    h = yaw_filter(lid[:, [6]] + np.arctan2(pose[1, 0], pose[0, 0]))
    world = np.concatenate([c[:, :3], lid[:, 3:6], h], 1)
    return lid, score, cls, kept, world


def track_sequence(boxes, counts, poses, cfg):
    """One sequence: boxes (F, K, 9) f32 lidar rows [x, y, z, dx, dy, dz, heading, score, label 1..3], counts (F), poses (F, 4, 4).
    Returns {'tracks': {id: {'boxes_global' (n, 9) f64, 'cls', 'score' (n), 'hit' (n), 'frame' (n), 'state'}} (post-processed),
    'kept': [per-frame bool mask of the overlap filter], 'margin': Margin}"""
    margin = Margin()
    F = len(counts)
    frames = [preprocess(boxes[f], int(counts[f]), np.asarray(poses[f], np.float64), cfg, margin) for f in range(F)]
    det = [(fr[1][fr[3]], fr[2][fr[3]], fr[4][fr[3]]) for fr in frames]          # score, cls, world of the kept rows
    s1, s2, mthr = cfg['FIRST_STAGE_THRESHOLD'], cfg['SECOND_STAGE_THRESHOLD'], cfg['MERGE_THRESHOLD']
    sthr = np.asarray(cfg['SCORE_THRESHOLD'], np.float64)
    entries = {}                                       # id -> list of (frame, box, cls, score, hit)
    tracks, next_id = [], 0
    for f in range(F):
        score, cls, world = det[f]
        tkb = np.array([t.predict(f, margin)[:9] for t in tracks], np.float32).reshape(-1, 9)
        tkc = np.array([t.cls for t in tracks], np.int64)
        if not tracks:
            births = np.arange(len(score))
        else:
            hi = np.flatnonzero(score >= sthr[cls - 1])
            lo = np.flatnonzero(~(score >= sthr[cls - 1]))
            ok, aff = _affinity(tkb, tkc, world[hi], cls[hi], s1, margin, 'stage 1 iou')
            m1 = _assign(ok, aff, margin, 'stage 1')
            for ti, di in m1:
                tracks[ti].update(world[hi[di]], cls[hi[di]], score[hi[di]], False)
            left = np.setdiff1d(np.arange(len(tracks)), m1[:, 0])
            ok, aff = _affinity(tkb[left], tkc[left], world[lo], cls[lo], s2, margin, 'stage 2 iou')
            for ti, di in _assign(ok, aff, margin, 'stage 2'):
                tracks[left[ti]].update(world[lo[di]], cls[lo[di]], score[lo[di]], True)
            births = np.setdiff1d(hi, hi[m1[:, 1]])
        for di in births:
            tracks.append(_Track(world[di], cls[di], score[di], f, next_id, cfg, cfg['FILTER']['DELTA_T']))
            next_id += 1
        dep = _merge([t.bbox for t in tracks], np.array([t.cls for t in tracks], np.int64), np.array([t.id for t in tracks]),
                     mthr, margin)
        for j in reversed(dep):
            tracks.pop(j)
        for t in tracks:
            entries.setdefault(t.id, []).append((f, np.asarray(t.bbox, np.float64).copy(), t.cls, t.score, t.hit))
    # reverse pass
    by_frame = [[] for _ in range(F)]
    for tid in sorted(entries):
        for k, e in enumerate(entries[tid]):
            by_frame[e[0]].append((tid, k == 0, e))
    rev = []
    for f in range(F - 1, -1, -1):
        score, cls, world = det[f]
        rb = [t.predict(f, margin)[:9] for t in rev]
        rc = [t.cls for t in rev]
        for tid, start, e in by_frame[f]:
            if not start:
                rb.append(e[1][:9])
                rc.append(e[2])
        rb, rc = np.array(rb, np.float32).reshape(-1, 9), np.array(rc, np.int64)
        if len(rb):
            lo = np.flatnonzero(~(score >= sthr[cls - 1]))
            ok, aff = _affinity(rb, rc, world[lo], cls[lo], s2, margin, 'reverse iou')
            for ti, di in _assign(ok, aff, margin, 'reverse'):
                if ti < len(rev):
                    rev[ti].update(world[lo[di]], cls[lo[di]], score[lo[di]], True)
        dep = _merge([t.bbox for t in rev], np.array([t.cls for t in rev], np.int64), np.array([t.id for t in rev]), mthr, margin)
        for j in reversed(dep):
            rev.pop(j)
        for t in rev:
            entries[t.id].insert(0, (f, np.asarray(t.bbox, np.float64).copy(), t.cls, t.score, t.hit))
        for tid, start, e in by_frame[f]:
            if start:
                rev.append(_Track(e[1][:7], e[2], e[3], f, tid, cfg, -0.1))
    return {'tracks': post_process(entries, cfg, margin), 'kept': [fr[3] for fr in frames], 'margin': margin}


def post_process(entries, cfg, margin):
    """empty_track_delete, velocity_optimize, motion_classify, static_drift_eliminate"""
    out = {}
    for tid, es in entries.items():
        hit = np.array([e[4] for e in es])
        if np.sum(hit > 0) < cfg['LEAST_AGE']:
            continue
        pos = np.flatnonzero(hit > 0)
        es = es[pos[0]:pos[-1] + 1]
        boxes = np.stack([e[1] for e in es])
        n, hl = len(es), cfg['HEADER_LENGTH']
        for k in range(hl if n > hl else n - 1):
            boxes[k, 7:9] = (boxes[k + 1, :2] - boxes[k, :2]) * 10.
        hit = np.array([e[4] for e in es])
        h1 = np.flatnonzero(hit == 1)
        state = 'static'
        if len(h1) >= 2:
            b = boxes[h1, :7].astype(np.float32)
            far = _far(b, b)
            if far.any():                                    # two hit boxes apart: dynamic whatever the other pairs give
                state = 'dynamic'
            else:
                ov = boxes_overlap_bev(b, b)
                margin.add(ov[ov > 0], 1e-4, 'motion')
                if np.any(ov <= 1e-4):
                    state = 'dynamic'
        # static_drift_eliminate rewrites trailing hit == 0 boxes, of which END_REMOVE has left none
        out[tid] = {'boxes_global': boxes, 'cls': np.array([e[2] for e in es]), 'score': np.array([e[3] for e in es], np.float32),
                    'hit': hit, 'frame': np.array([e[0] for e in es]), 'state': state}
    return out


def check_device(res, s, ref):
    """Assert that sequence s of a detzero_b200.track.TrackResult takes every decision of ``ref`` (this module's track_sequence
    result, or the golden in the same form): the overlap filter's keep flags, the track ids, and per track its entry frames, hit
    flags, class and motion state.  Boxes agree within 5e-3 m (5e-2 m/s for the velocity) and 1e-4 rad, scores exactly."""
    kept = res.kept[s].cpu().numpy()
    for f, k in enumerate(ref['kept']):
        assert np.array_equal(kept[f, :len(k)], k), 'keep flags differ at frame %d' % f
    rows = res.tracks(s)
    assert [int(r[0]) for r in rows] == sorted(ref['tracks']), 'track ids differ'
    eb, es = res.ent_box[s].cpu().numpy(), res.ent_score[s].cpu().numpy()
    eh, ef = res.ent_hit[s].cpu().numpy(), res.ent_frame[s].cpu().numpy()
    for tid, cls, first, cnt, dyn, off in rows:
        t = ref['tracks'][int(tid)]
        sl = slice(off, off + cnt)
        assert np.array_equal(ef[sl], t['frame']), ('entry frames', tid)
        assert np.array_equal(eh[sl], t['hit']), ('hit flags', tid)
        assert cls == t['cls'][0] and bool(dyn) == (t['state'] == 'dynamic'), ('class / state', tid)
        b, rb = eb[sl], t['boxes_global']
        assert np.abs(b[:, :6] - rb[:, :6]).max() < 5e-3 and np.abs(b[:, 7:9] - rb[:, 7:9]).max() < 5e-2, ('boxes', tid)
        assert np.abs(np.angle(np.exp(1j * (b[:, 6] - rb[:, 6])))).max() < 1e-4, ('heading', tid)
        assert np.array_equal(es[sl], t['score']), ('scores', tid)

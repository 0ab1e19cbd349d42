"""Host restatement of CenterPoint test-time augmentation (TEST INFRASTRUCTURE): view expansion
(detection/detzero_det/datasets/augmentor/test_time_augmentor.py:9-100), box un-augmentation (CenterPoint.test_time_augment,
detection/detzero_det/models/centerpoint.py:131-208) and weighted_boxes_fusion_3d (utils/ensemble_utils/wbf_3d.py:10-190) with
the wbf_online settings.  Pinned against tests/golden/tta.npz, written by the reference's own code (make_golden_tta.py)."""
import numpy as np

from . import boxes_iou3d

IOU_THR = [0.8, 0.6, 0.7]
SKIP_BOX_THR = [0.1, 0.01, 0.01]


def view_ops(names):
    """[(op, param)] from the reference's view names: op in original / flip_x / flip_y / flip_xy / rot / scale"""
    out = []
    for n in names:
        if n == 'tta_original':
            out.append(('original', 0.0))
        else:
            _, kind, p = n.split('_', 2)
            out.append(('flip_' + p, 0.0) if kind == 'flip' else (kind, float(p)))
    return out


def _cos_sin(angle):
    import torch
    a = torch.tensor([float(angle)], dtype=torch.float64).float()
    return np.float32(torch.cos(a)[0]), np.float32(torch.sin(a)[0]), np.float32(a[0])


def _fma_f32(a, b, c):
    """round_f32(a*b + c) for float32 arrays: a*b is exact in float64; the float64 sum is rounded once more, which differs from
    a single rounding only when it lands exactly on a float32 midpoint -- asserted not to happen"""
    p = a.astype(np.float64) * b.astype(np.float64)
    t = p + c.astype(np.float64)
    bb = t - p
    err = (p - (t - bb)) + (c.astype(np.float64) - bb)            # exact error of the float64 sum
    r = t.astype(np.float32)
    mid = np.abs(t - r.astype(np.float64)) == 0.5 * np.spacing(np.abs(r)).astype(np.float64)
    assert not np.any(mid & (err != 0)), 'float32 midpoint in the float64 emulation of fma'
    return r


def rotate_xy(x, y, c, s):
    """rotate_points_along_z's float32 result ([x y] @ [[c s] [-s c]]): x' = fma(y, -s, x*c), y' = fma(y, c, x*s)"""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    c, s = np.float32(c), np.float32(s)
    return _fma_f32(y, np.full_like(y, -s), x * c), _fma_f32(y, np.full_like(y, c), x * s)


def augment(points, names):
    """points (N, 3+C) float32 of one frame -> list of V augmented copies (x, y, z changed, features kept)"""
    out = []
    for op, p in view_ops(names):
        q = np.array(points, dtype=np.float32, copy=True)
        if op == 'flip_x':
            q[:, 1] = -q[:, 1]
        elif op == 'flip_y':
            q[:, 0] = -q[:, 0]
        elif op == 'flip_xy':
            q[:, 0] = -q[:, 0]; q[:, 1] = -q[:, 1]
        elif op == 'rot':
            c, s, _ = _cos_sin(p)
            q[:, 0], q[:, 1] = rotate_xy(q[:, 0], q[:, 1], c, s)
        elif op == 'scale':
            q[:, :3] *= np.float32(p)
        out.append(q)
    return out


def unaugment(boxes, names):
    """boxes (V, K, 7+) float32, view v in view v's frame -> float32 boxes in the original frame"""
    b = np.array(boxes, dtype=np.float32, copy=True)
    pi = np.float32(np.pi)
    for v, (op, p) in enumerate(view_ops(names)):
        x = b[v]
        if op == 'flip_x':
            x[:, 1] = -x[:, 1]; x[:, 6] = -x[:, 6]
        elif op == 'flip_y':
            x[:, 0] = -x[:, 0]; x[:, 6] = -(x[:, 6] + pi)
        elif op == 'flip_xy':
            x[:, 0:2] = -x[:, 0:2]; x[:, 6] = x[:, 6] + pi
        elif op == 'rot':
            c, s, a = _cos_sin(-p)
            x[:, 0], x[:, 1] = rotate_xy(x[:, 0], x[:, 1], c, s)
            x[:, 6] = x[:, 6] + a
        elif op == 'scale':
            x[:, :6] = x[:, :6] / np.float32(p)
    return b


def wbf_3d(boxes, scores, labels, iou_thr=IOU_THR, skip_box_thr=SKIP_BOX_THR):
    """weighted_boxes_fusion_3d(conf_type='avg', iou_type='3d', unit weights, allows_overflow=False).
    boxes (V, K, 7), scores (V, K), labels (V, K) (label 0 = padding).  Ties: score descending, then (view, row) ascending.
    Returns dict: boxes (M, 7) f32, scores (M,) f64, labels (M,), members (list of (view, row) lists), min_margin
    (smallest |best IoU - thr| over the clustering decisions)."""
    V, K = boxes.shape[0], boxes.shape[1]
    boxes = np.asarray(boxes, np.float32)
    scores = np.asarray(scores, np.float32).reshape(V, K)
    labels = np.asarray(labels).reshape(V, K).astype(np.int64)
    clusters, margin = [], np.inf
    for lab in sorted(set(labels[labels > 0].tolist())):
        if lab > len(iou_thr):
            continue
        vv, rr = np.nonzero(labels == lab)
        idx = vv * K + rr
        sc = scores[vv, rr].astype(np.float64)
        order = np.lexsort((idx, -sc))
        order = order[sc[order] >= skip_box_thr[lab - 1]]
        fused, acc, conf, members = [], [], [], []
        for o in order:
            v, r, s = int(vv[o]), int(rr[o]), float(sc[o])
            b = boxes[v, r, :7]
            best, bi = -1.0, -1
            if fused:
                ious = boxes_iou3d(b[None], np.asarray(fused, np.float32))[0]
                bi = int(np.argmax(ious))
                best = float(ious[bi])
            margin = min(margin, abs(max(best, 0.0) - iou_thr[lab - 1]))
            if bi >= 0 and best > iou_thr[lab - 1]:
                a = acc[bi]
                a[:] = (a.astype(np.float64) + s * b.astype(np.float64)).astype(np.float32)
                conf[bi] += s
                members[bi].append((v, r))
                f = (a.astype(np.float64) / conf[bi]).astype(np.float32)
                f[6] = fused[bi][6]
                fused[bi] = f
            else:
                fused.append(b.copy())
                acc.append((s * b.astype(np.float64)).astype(np.float32))
                conf.append(s)
                members.append([(v, r)])
        for f, c, m in zip(fused, conf, members):
            n = len(m)
            if n == 1:
                score = c / V
            else:
                w1 = np.float32(c / n)
                score = float(np.float32((np.float64(np.float32(w1 * np.float32(n))) / V) if n < V else (np.float64(w1) * V) / V))
            clusters.append((score, m[0][0] * K + m[0][1], f, lab, m))
    clusters.sort(key=lambda t: (-t[0], t[1]))
    return {'boxes': np.asarray([c[2] for c in clusters], np.float32).reshape(-1, 7),
            'scores': np.asarray([c[0] for c in clusters], np.float64),
            'labels': np.asarray([c[3] for c in clusters], np.int64),
            'members': [c[4] for c in clusters], 'min_margin': margin}

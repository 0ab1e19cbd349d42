"""Seeded synthetic weights and the default CenterPoint model config for benchmarks, smoke runs and parity tests.

There are no released checkpoints on disk (SURVEY.md §8c): product modules, the oracle and the reference modules (when
golden vectors are generated) are all filled from the SAME seeded function of (key name, shape) -- identical key names
=> identical tensors, regardless of how each side constructs its module tree.  BatchNorm running stats are randomised
away from (0, 1) so that folding errors show.  Lives in the package so that bench.py's GPU arm does not need ``oracle/``
or ``tests/`` on its import path."""
import zlib

import numpy as np
import torch

from .config import AttrDict

#: sparse-conv arithmetic of the shipped config / bench / smoke (detzero_b200/_lib.py MODES), and the per-mode bound on the
#: backbone output features vs the fp32 oracle (relative to max |feature|) that the parity tests enforce
DEFAULT_SP_MODE = 'bf16x2'
SP_MODE_TOL = {'fp32': 2e-5, 'tf32x3': 2e-4, 'bf16x2': 2e-4, 'tf32': 5e-3, 'bf16': 3e-2}

def _rng(seed, key):
    return np.random.default_rng([int(seed), zlib.crc32(key.encode())])


def seeded_tensor(key, shape, seed, kind=None):
    shape = tuple(int(s) for s in shape)
    g = _rng(seed, key)
    leaf = key.split('.')[-1]
    if '.hm.' in key and leaf == 'bias' and len(shape) == 1 and kind is None and key.endswith('.1.bias'):
        return torch.from_numpy((-2.19 + g.normal(0, 0.05, shape)).astype(np.float32))     # center_head.py:33 init
    if '.hm.' in key and key.endswith('.1.weight'):
        fan_in = max(1, int(np.prod(shape)) // max(1, shape[0]))
        return torch.from_numpy((g.normal(0, 0.15 * np.sqrt(2.0 / fan_in), shape)).astype(np.float32))
    if leaf == 'num_batches_tracked':
        return torch.zeros(shape, dtype=torch.long)
    if leaf == 'running_var':
        a = g.uniform(0.5, 1.5, shape)
    elif leaf == 'running_mean':
        a = g.normal(0, 0.1, shape)
    elif leaf == 'bias' or leaf == 'in_proj_bias':
        a = g.normal(0, 0.05, shape)
    elif leaf == 'weight' and len(shape) == 1:           # norm scale
        a = g.uniform(0.5, 1.5, shape)
    else:                                                # conv / linear weight: He-style, fan_in = prod(shape[1:])...
        fan_in = max(1, int(np.prod(shape)) // max(1, shape[0]))
        a = g.normal(0, np.sqrt(2.0 / fan_in), shape)
    return torch.from_numpy(np.asarray(a, dtype=np.float32).reshape(shape))


def seeded_state_dict(module, seed):
    """state_dict with every entry replaced by its seeded value (same dtype/shape)"""
    sd = module.state_dict()
    out = {}
    for k in sd:
        t = seeded_tensor(k, sd[k].shape, seed)
        out[k] = t.to(sd[k].dtype) if sd[k].dtype != torch.long else t
    return out


def load_seeded(module, seed):
    sd = seeded_state_dict(module, seed)
    module.load_state_dict(sd)
    return sd



def model_cfg(backbone='VoxelResBackBone8x', mode='fp32', channels=None):
    cfg = AttrDict({
        'NAME': 'CenterPoint', 'SECOND_STAGE': False,
        'VFE': {'NAME': 'MeanVFE'},
        'BACKBONE_3D': {'NAME': backbone, 'COMPUTE_MODE': mode},
        'MAP_TO_BEV': {'NAME': 'HeightCompression', 'NUM_BEV_FEATURES': 256},
        'BACKBONE_2D': {'NAME': 'BaseBEVBackbone', 'LAYER_NUMS': [5, 5], 'LAYER_STRIDES': [1, 2],
                        'NUM_FILTERS': [128, 256], 'UPSAMPLE_STRIDES': [1, 2], 'NUM_UPSAMPLE_FILTERS': [256, 256],
                        'COMPUTE_MODE': mode},
        'DENSE_HEAD': {
            'NAME': 'CenterHead', 'CLASS_AGNOSTIC': False, 'COMPUTE_MODE': mode,
            'CLASS_NAMES_EACH_HEAD': [['Vehicle', 'Pedestrian', 'Cyclist']],
            'SHARED_CONV_CHANNEL': 64, 'USE_BIAS_BEFORE_NORM': True, 'NUM_HM_CONV': 2, 'IOU_WEIGHT': 1,
            'SEPARATE_HEAD_CFG': {
                'HEAD_ORDER': ['center', 'center_z', 'dim', 'rot', 'iou'],
                'HEAD_DICT': {'center': {'out_channels': 2, 'num_conv': 2}, 'center_z': {'out_channels': 1, 'num_conv': 2},
                              'dim': {'out_channels': 3, 'num_conv': 2}, 'rot': {'out_channels': 2, 'num_conv': 2},
                              'iou': {'out_channels': 1, 'num_conv': 2}}},
            'TARGET_ASSIGNER_CONFIG': {'FEATURE_MAP_STRIDE': 8, 'NUM_MAX_OBJS': 500, 'GAUSSIAN_OVERLAP': 0.1, 'MIN_RADIUS': 2},
            'POST_PROCESSING': {'SCORE_THRESH': 0.03, 'POST_CENTER_LIMIT_RANGE': [-80, -80, -10.0, 80, 80, 10.0],
                                'MAX_OBJ_PER_SAMPLE': 500,
                                'NMS_CONFIG': {'NMS_TYPE': 'nms_gpu', 'NMS_THRESH': 0.7, 'NMS_PRE_MAXSIZE': 4096,
                                               'NMS_POST_MAXSIZE': 500}}},
        'POST_PROCESSING': {'RECALL_THRESH_LIST': [0.3, 0.5, 0.7], 'SCORE_THRESH': 0.03, 'OUTPUT_RAW_SCORE': False,
                            'EVAL_METRIC': 'waymo'},
    })
    if channels is not None:
        cfg.BACKBONE_3D.CHANNELS = channels
    return cfg


CLASS_NAMES = ['Vehicle', 'Pedestrian', 'Cyclist']


# ---- refiner: the REGRESSION sections of the shipped configs (refining/tools/cfgs/ref_model_cfgs/vehicle_{prm,grm,crm}_model.yaml)
# ---- and seeded inputs of the reference's shapes (SURVEY.md Appendix B)
def prm_cfg():
    return AttrDict({'NAME': 'PositionTransformer', 'QUERY_ENCODER': [128, 128], 'MEMORY_ENCODER': [128, 128], 'REGRESSION_MLP': [512],
                     'DECODER': {'NAME': 'PositionHead', 'num_classes': 3, 'num_heads': 8, 'num_decoder_layers': 1, 'auxiliary': True,
                                 'cross_only': False, 'hidden_channel': 256, 'dropout': 0.1, 'bn_momentum': 0.1, 'activation': 'relu',
                                 'ffn_channel': 256},
                     'LOSS_CLS': {'type': 'CrossEntropyLoss', 'reduction': 'mean', 'ignore_index': -1}})


def grm_cfg():
    return AttrDict({'NAME': 'GeometryTransformer', 'QUERY_ENCODER': [128, 128], 'MEMORY_ENCODER': [128, 128], 'REGRESSION_MLP': [512],
                     'EMBED_DIMS': 256, 'ANCHOR_SIZES': [[4.8, 1.8, 1.5], [10.0, 2.6, 3.2], [2.0, 1.0, 1.6]],
                     'DECODER': {'NAME': 'GeometryHead', 'num_classes': 3, 'num_heads': 8, 'num_decoder_layers': 1, 'auxiliary': True,
                                 'cross_only': False, 'memory_self_attn': False, 'hidden_channel': 256, 'ffn_channel': 256,
                                 'dropout': 0.1, 'bn_momentum': 0.1, 'activation': 'relu'}})


def crm_cfg():
    return AttrDict({'NAME': 'ConfidencePointnet', 'ENCODER_MLP': [128, 128], 'REGRESSION_MLP': [512], 'SCORE_THRESH': [0.35, 0.7]})


def refine_models(seed, mode='fp32', classes=CLASS_NAMES, device='cuda'):
    """{class: {'PRM', 'GRM', 'CRM': refine.RefineTemplate}} of the shipped REGRESSION configs with seeded weights (distinct per class
    and kind), as offboard.refine_sequence takes them"""
    from .refine import RefineTemplate
    out = {}
    for i, c in enumerate(classes):
        out[c] = {}
        for j, (kind, name, cfg, qd, md) in enumerate((('PRM', 'PositionRefineModel', prm_cfg(), 32, 32),
                                                       ('GRM', 'GeometryRefineModel', grm_cfg(), 11, 4),
                                                       ('CRM', 'ConfidenceRefineModel', crm_cfg(), 32, 32))):
            cfg.COMPUTE_MODE = mode
            m = RefineTemplate(AttrDict({'NAME': name, 'QUERY_POINT_DIMS': qd, 'MEMORY_POINT_DIMS': md, 'REGRESSION': cfg})).eval()
            load_seeded(m, int(seed) * 16 + 3 * i + j)
            out[c][kind] = m.to(device)
    return out


def prm_inputs(seed, B=2, boxes=200, qpts=256, mpts=48, dims=32):
    g = np.random.default_rng(seed)
    box_num = g.integers(20, boxes + 1, B)
    box_num[0] = boxes                                   # one full track
    mask = np.zeros((B, boxes), np.float32)
    for b in range(B):
        mask[b, box_num[b]:] = 1
    return {'pos_query_points': torch.from_numpy(g.normal(0, 1, (B, boxes, qpts, dims)).astype(np.float32)),
            'pos_memory_points': torch.from_numpy(g.normal(0, 1, (B, boxes, mpts, dims)).astype(np.float32)),
            'pos_trajectory': torch.from_numpy(g.normal(0, 2, (B, boxes, 7)).astype(np.float32)),
            'padding_mask': torch.from_numpy(mask)}


def grm_inputs(seed, B=2, mem=4096, q=3, qpts=256):
    g = np.random.default_rng(seed)
    return {'geo_memory_points': torch.from_numpy(g.normal(0, 1, (B, mem, 11)).astype(np.float32)),
            'geo_query_points': torch.from_numpy(g.normal(0, 1, (B, q, qpts, 4)).astype(np.float32)),
            'geo_query_boxes': torch.from_numpy(g.normal(0, 1, (B, q, 7)).astype(np.float32)),
            'geo_query_num': torch.tensor([q] + [max(1, q - 1)] * (B - 1))}


def crm_inputs(seed, B=2, boxes=200, pts=256, dims=32):
    g = np.random.default_rng(seed)
    return {'conf_points': torch.from_numpy(g.normal(0, 1, (B, boxes, pts, dims)).astype(np.float32))}


# ---- a tracked sequence for the refiner input builder (detzero_b200/refine/data.py)
def _rz(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def synthetic_sequence(seed, frames=20, tracks=8, L=200, n_background=20000, max_pts=3000, origin=(5000.0, -3000.0, 50.0),
                       min_len=1, enlarge=1.1, margin=1e-3, ego_step=1.0, max_speed=0.4, lengths=None, cls=None,
                       radius=45.0):
    """A seeded tracked sequence: ego poses with world translations around ``origin`` (about 5 km) and yaw wrapping through +-pi,
    objects moving on smooth paths (headings wrapping too), 0..~max_pts points on and inside each box over a synth_waymo_cloud
    background, and no point within ``margin`` of any enlarged box face, so crop membership is unambiguous.
    Returns a dict: frames (N, 6) f32 collated rows [b=frame, x, y, z, tanh(i), elongation] in the lidar frame, frame_offsets (F+1),
    poses (F, 4, 4) f64, and the TrackBatch fields as numpy arrays (boxes (B, L, 7) f64 world, frame_of_box, scores, box_num, cls,
    track_uid).  ``lengths`` / ``cls`` fix the box count / class of each track (default: random); each track starts 6 m to
    ``radius`` m from the ego."""
    from .det.dataset import synth_waymo_cloud
    g = np.random.default_rng([int(seed), 0x5E9])
    F = int(frames)
    yaw0 = np.pi - 0.4
    ego_yaw = yaw0 + 0.8 * np.arange(F) / max(F - 1, 1)
    ego_xy = np.cumsum(np.stack([np.cos(ego_yaw), np.sin(ego_yaw)], 1) * ego_step, 0)
    poses = np.zeros((F, 4, 4))
    for f in range(F):
        tilt = np.array([[1, 0, 0], [0, np.cos(0.004), -np.sin(0.004)], [0, np.sin(0.004), np.cos(0.004)]])
        poses[f, :3, :3] = _rz(ego_yaw[f]) @ tilt
        poses[f, :3, 3] = np.asarray(origin) + [ego_xy[f, 0], ego_xy[f, 1], 0.01 * f]
        poses[f, 3, 3] = 1
    B = int(tracks)
    boxes = np.zeros((B, L, 7))
    fob = np.zeros((B, L), np.int32)
    scores = np.zeros((B, L), np.float32)
    box_num = np.zeros(B, np.int32)
    cls = (g.integers(1, 4, B) if cls is None else np.asarray(cls)).astype(np.int32)
    dims_by_cls = np.array([[4.7, 2.0, 1.6], [0.9, 0.9, 1.8], [1.9, 0.8, 1.7]])
    obj_pts = [[] for _ in range(F)]
    frame_boxes = [[] for _ in range(F)]
    for b in range(B):
        n = int(g.integers(min(min_len, F), min(L, F) + 1)) if lengths is None else int(lengths[b])
        start = int(g.integers(0, F - n + 1))
        box_num[b] = n
        dims = dims_by_cls[cls[b] - 1] * g.uniform(0.9, 1.1, 3)
        r0, a0 = g.uniform(6, radius), g.uniform(-np.pi, np.pi)
        c0 = poses[start, :3, 3] + [r0 * np.cos(a0), r0 * np.sin(a0), -1.2]
        h0, speed, turn = g.uniform(-np.pi, np.pi), g.uniform(0, max_speed), g.uniform(-0.05, 0.05)
        pts_n = np.where(g.random(n) < 0.1, 0, np.exp(g.uniform(0, np.log(max_pts), n)).astype(int))
        for j in range(n):
            f = start + j
            h = h0 + turn * j
            c = c0 + speed * j * np.array([np.cos(h), np.sin(h), 0.0]) + poses[f, :3, 3] - poses[start, :3, 3]
            boxes[b, j] = [c[0], c[1], c[2], dims[0], dims[1], dims[2], h]
            fob[b, j] = f
            scores[b, j] = np.float32(g.uniform(0.05, 0.95))
            u = g.uniform(-0.48, 0.48, (pts_n[j], 3)) * dims                       # inside the (unenlarged) box
            u[: pts_n[j] // 3, 2] = -dims[2] / 2 + 0.02                            # some on the bottom face
            w = u @ _rz(h).T + c
            obj_pts[f].append(np.concatenate([w, g.uniform(0, 1, (len(w), 1))], 1))
            frame_boxes[f].append(boxes[b, j])
    rows, offsets = [], [0]
    from scipy.spatial import cKDTree
    for f in range(F):
        bg = synth_waymo_cloud(seed=int(seed) * 1000 + f, n_target=n_background)
        P = poses[f]
        bgw = np.concatenate([bg[:, :3].astype(np.float64) @ P[:3, :3].T + P[:3, 3], bg[:, 3:4]], 1)
        pw = np.concatenate([bgw] + obj_pts[f], 0) if obj_pts[f] else bgw
        keep = np.ones(len(pw), bool)
        if frame_boxes[f]:
            fb = np.array(frame_boxes[f])
            tree = cKDTree(pw[:, :2])
            for bx, idx in zip(fb, tree.query_ball_point(fb[:, :2], np.linalg.norm(fb[:, 3:5] * enlarge, axis=1) / 2 + 0.1)):
                idx = np.asarray(idx, np.int64)
                if not len(idx):
                    continue
                rel = (pw[idx, :3] - bx[:3]) @ _rz(bx[6])                          # box frame
                half = bx[3:6] * enlarge / 2
                d = np.abs(rel) - half
                outside = np.max(d, 1)
                keep[idx[np.abs(outside) < margin * 3]] = False                   # within a few margins of an enlarged face
        pw = pw[keep]
        loc = ((pw[:, :3] - P[:3, 3]) @ P[:3, :3]).astype(np.float32)
        r = np.zeros((len(pw), 6), np.float32)
        r[:, 0], r[:, 1:4], r[:, 4], r[:, 5] = f, loc, np.tanh(pw[:, 3]), 0.0
        rows.append(r)
        offsets.append(offsets[-1] + len(r))
    return {'frames': np.concatenate(rows, 0), 'frame_offsets': np.asarray(offsets, np.int64), 'poses': poses, 'boxes': boxes,
            'frame_of_box': fob, 'scores': scores, 'box_num': box_num, 'cls': cls,
            'track_uid': (np.arange(B, dtype=np.int64) * 7919 + int(seed) * 104729 + 1)}


def detections_from_sequence(s, seed, miss=0.1, fp=10, K=500):
    """Gathered lidar detections (F, K, 9) of a synthetic_sequence's ground-truth boxes, for the tracker: 3 cm / 0.01 rad / 0.5 %
    jitter, about ``miss`` of the boxes missed (never the first or last two of a track), ``fp`` far false positives per frame, rows
    shuffled.  Returns boxes, counts (F), gt (F, K) (the ground-truth track of each row, -1 for a false positive)."""
    g = np.random.default_rng([int(seed), 0xC0B])
    F = len(s['poses'])
    dims = [[4.7, 2.0, 1.6], [0.9, 0.9, 1.8], [1.9, 0.8, 1.7]]
    rows = [[] for _ in range(F)]
    for b in range(len(s['box_num'])):
        n = int(s['box_num'][b])
        for j in range(n):
            if 2 <= j < n - 2 and g.random() < miss:
                continue
            f = int(s['frame_of_box'][b, j])
            P, w = s['poses'][f], s['boxes'][b, j]
            loc = (w[:3] + g.normal(0, 0.03, 3) - P[:3, 3]) @ P[:3, :3]
            h = w[6] + g.normal(0, 0.01) - np.arctan2(P[1, 0], P[0, 0])
            rows[f].append(([*loc, *(w[3:6] * (1 + g.normal(0, 0.005, 3))), np.arctan2(np.sin(h), np.cos(h)),
                             g.uniform(0.3, 0.95), s['cls'][b]], b))
    for f in range(F):
        for _ in range(fp):
            a, r, c = g.uniform(-np.pi, np.pi), g.uniform(300, 500), int(g.integers(1, 4))
            rows[f].append(([r * np.cos(a), r * np.sin(a), -1.0, *dims[c - 1], g.uniform(-np.pi, np.pi), g.uniform(0.02, 0.3), c], -1))
    boxes, gt, counts = np.zeros((F, K, 9), np.float32), np.full((F, K), -1), np.zeros(F, np.int32)
    for f in range(F):
        if len(rows[f]) > K:
            raise ValueError('frame %d has %d detections (K = %d)' % (f, len(rows[f]), K))
        for i, k in enumerate(g.permutation(len(rows[f]))):
            boxes[f, i], gt[f, i] = rows[f][k]
        counts[f] = len(rows[f])
    return boxes, counts, gt


def synthetic_detections(seed, frames=199, objects=300, false_positives=40, K=500, miss=0.1, chain=0, origin=(5000.0, -3000.0, 50.0)):
    """Seeded gathered detections of one sequence for the tracker, laid out so that no association, merge or overlap-filter decision
    sits near its threshold: objects drive in lanes 12 m apart (one class and speed per lane: parked, slow and fast vehicles,
    pedestrians, cyclists), 30 / 10 / 5 m apart within a lane, each alive over a random run of frames, detected with 3 cm / 0.01 rad
    jitter, dropped with probability ``miss``, and with one low-score stretch (score < 0.1) each; ``false_positives`` boxes per frame
    far from every lane, one in ten above the score threshold; ``chain`` static pedestrians 0.73 m apart without jitter, so that
    each detection overlaps three tracks (one large association component).  The ego drives through the scene.
    Returns boxes (F, K, 9) f32 lidar rows [x, y, z, dx, dy, dz, heading, score, label], counts (F), poses (F, 4, 4) and the ground
    truth gt_id (F, K) (-1 for a false positive)."""
    g = np.random.default_rng([int(seed), 0x7AC])
    F = int(frames)
    yaw = 0.3 + 0.2 * np.arange(F) / max(F - 1, 1)
    poses = np.zeros((F, 4, 4))
    for f in range(F):
        poses[f, :3, :3] = _rz(yaw[f])
        poses[f, :3, 3] = np.asarray(origin) + [2.0 * f, 0.5 * f, 0.0]
        poses[f, 3, 3] = 1
    kinds = [(1, 0.0, 30.), (1, 1.0, 30.), (1, 10.0, 30.), (2, 1.2, 5.), (3, 4.0, 10.)]     # class, speed, spacing
    dims_by_cls = np.array([[4.7, 2.0, 1.6], [0.9, 0.6, 1.8], [1.9, 0.8, 1.7]])
    dets = [[] for _ in range(F)]
    lane, placed = 0, 0
    while placed < objects:
        cls, speed, gap = kinds[lane % len(kinds)]
        direction = 1.0 if lane % 2 == 0 else -1.0
        for k in range(min(8, objects - placed)):
            start = int(g.integers(0, max(F - 8, 1)))
            end = int(g.integers(min(start + 8, F), F + 1))
            dims = dims_by_cls[cls - 1] * g.uniform(0.95, 1.05, 3)
            low0 = int(g.integers(start, end))
            low1 = low0 + int(g.integers(1, 4))
            x0 = k * gap * 1.2 + g.uniform(0, 0.2 * gap) - 120.
            for f in range(start, end):
                if g.random() < miss:
                    continue
                c = np.array([x0 + direction * speed * 0.1 * f, 12.0 * lane - 60., -1.0]) + g.normal(0, 0.03, 3)
                h = (0.0 if direction > 0 else np.pi - 1e-3) + g.normal(0, 0.01)
                sc = g.uniform(0.02, 0.09) if low0 <= f < low1 else g.uniform(0.3, 0.95)
                dets[f].append((c, dims * (1 + g.normal(0, 0.005, 3)), h, sc, cls, placed + k))
        placed += min(8, objects - placed)
        lane += 1
    for k in range(chain):
        for f in range(F):
            dets[f].append((np.array([-150. + 0.73 * k, -90., -1.0]), dims_by_cls[1], 0.0, 0.8, 2, objects + k))
    for f in range(F):
        for _ in range(int(false_positives)):
            c = np.array([g.uniform(-600, 600), g.uniform(300, 900), -1.0])
            cls = int(g.integers(1, 4))
            sc = g.uniform(0.1, 0.3) if g.random() < 0.1 else g.uniform(0.01, 0.09)
            dets[f].append((c, dims_by_cls[cls - 1], g.uniform(-np.pi, np.pi), sc, cls, -1))
    boxes = np.zeros((F, K, 9), np.float32)
    gt_id = np.full((F, K), -1, np.int64)
    counts = np.zeros(F, np.int32)
    for f in range(F):
        order = g.permutation(len(dets[f]))[:K]
        R, t = poses[f, :3, :3], poses[f, :3, 3]
        for i, j in enumerate(order):
            c, d, h, sc, cls, gid = dets[f][j]
            lw = (np.asarray(origin) + c - t) @ R                               # c is relative to the origin
            hl = h - yaw[f]
            boxes[f, i] = [*lw, *d, np.arctan2(np.sin(hl), np.cos(hl)), sc, cls]
            gt_id[f, i] = gid
        counts[f] = len(order)
    return {'boxes': boxes, 'counts': counts, 'poses': poses, 'gt_id': gt_id}

"""The PRM's position targets (refine.modules.TargetAssigner.encode_torch, mode 'position'; target_assign.py:32-53) on the host:
the reference's arithmetic, and the heading bin kept in 0..11 at built ties (yaw = -pi, the float32 neighbours of pi, the bin
edges and theirs), where the reference's floor gives 12 for +pi and the float32 headings just below it."""
import numpy as np
import torch

from detzero_b200.refine.modules import TargetAssigner

PI32 = np.float32(np.pi)                     # 3.14159274 > pi


def _ties():
    """float32 headings: -pi and +pi as float32 and their neighbours, every bin edge k pi / 6 - pi and its two neighbours, and a
    few folded values outside [-pi, pi]"""
    v = [-PI32, np.nextafter(-PI32, np.float32(0)), PI32, np.nextafter(PI32, np.float32(0)),
         np.nextafter(np.nextafter(PI32, np.float32(0)), np.float32(0)), np.float32(0)]
    for k in range(13):
        e = np.float32(k * np.pi / 6 - np.pi)
        v += [e, np.nextafter(e, np.float32(-4)), np.nextafter(e, np.float32(4))]
    v += [np.float32(3.5), np.float32(-3.5), np.nextafter(-PI32, np.float32(-4))]
    return np.array(v, np.float32)


def _encode(yaw):
    n = len(yaw)
    traj = torch.zeros((1, n, 7))
    traj[0, :, :3] = torch.arange(3 * n, dtype=torch.float32).reshape(n, 3) * 0.1
    gt = traj.clone()
    gt[0, :, :3] += 0.25
    gt[0, :, 6] = torch.from_numpy(yaw)
    data = {'pos_trajectory': traj, 'gt_pos_trajectory': gt, 'box_num': torch.tensor([n])}
    return TargetAssigner(mode='position').encode_torch(data), traj, gt


def _reference(traj, gt):
    """target_assign.py:32-53 as written (float32 tensors, the unclamped bin)"""
    traj_gt = gt.clone()
    idx = torch.where(traj_gt[:, :, 6] < -torch.pi)
    traj_gt[:, :, 6][idx] += 2 * torch.pi
    idx = torch.where(traj_gt[:, :, 6] > torch.pi)
    traj_gt[:, :, 6][idx] -= 2 * torch.pi
    anchors = (torch.arange(12, dtype=torch.float) * (2 * np.pi / 12) - np.pi)[None, None]
    return {'center_reg': traj_gt[:, :, :3] - traj[:, :, :3],
            'heading_reg': (traj_gt[:, :, 6:7].repeat(1, 1, 12) - anchors) / (np.pi / 12),
            'heading_cls': torch.floor((traj_gt[:, :, 6] + np.pi) / (np.pi / 6.)).long(), 'boxes_gt': traj_gt}


def test_position_targets_are_the_reference_with_the_bin_in_range():
    yaw = _ties()
    t, traj, gt = _encode(yaw)
    r = _reference(traj, gt)
    for k in ('center_reg', 'heading_reg', 'boxes_gt'):
        assert torch.equal(t[k], r[k]), k
    cls, rc = t['heading_cls'][0].numpy(), r['heading_cls'][0].numpy()
    assert cls.min() >= 0 and cls.max() <= 11
    assert (rc == 12).any(), 'the ties must reach the reference bin that does not exist'
    assert np.array_equal(cls, np.where(rc == 12, 11, rc))
    assert int(t['box_num'][0]) == len(yaw)


def test_heading_bin_at_the_ties():
    yaw = _ties()
    t, _, _ = _encode(yaw)
    cls = t['heading_cls'][0].numpy()
    h = t['boxes_gt'][0, :, 6].numpy().astype(np.float64)
    at = {float(y): int(c) for y, c in zip(yaw, cls)}
    assert at[float(-PI32)] == 0 and at[float(PI32)] == 11
    assert at[float(np.nextafter(PI32, np.float32(0)))] == 11
    # each heading lies in its bin [anchor, anchor + pi / 6), up to float32 rounding of the edge
    lo = cls * np.pi / 6 - np.pi
    assert (h >= lo - 1e-6).all() and (h <= lo + np.pi / 6 + 1e-6).all()
    assert (h >= -np.pi - 1e-6).all() and (h <= np.pi + 1e-6).all()


def test_cross_entropy_accepts_every_bin():
    t, _, _ = _encode(_ties())
    logits = torch.zeros((t['heading_cls'].numel(), 12))
    assert torch.isfinite(torch.nn.functional.cross_entropy(logits, t['heading_cls'].reshape(-1)))

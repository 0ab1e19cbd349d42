"""Golden vectors for the two host-side restatements pinned by tests/test_host_logic.py and tests/test_oracle.py, produced by the
reference's own code (needs the reference checkout, path as the first argument):
  * merge_sweeps.npz: DatasetTemplate.merge_sweeps (detection/detzero_det/datasets/dataset.py), its statements executed as they are;
  * iou_bev.npz: the rotated-BEV IoU of utils/detzero_utils/ops/iou3d_nms/src/iou3d_cpu.cpp, compiled by oracle/build_ref.py.

    python tests/golden/make_golden_host.py /path/to/reference
"""
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))


def merge_sweeps_inputs():
    g = np.random.default_rng(3)

    def pose():
        a = g.uniform(-0.2, 0.2)
        p = np.eye(4); p[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]; p[:3, 3] = g.uniform(-3, 3, 3)
        return p
    infos = [{'pose': pose(), 'time_stamp': 1550000000000000 - 100000 * k} for k in range(3)]
    pts = []
    for k in range(3):
        a = g.normal(0, 20, (500, 6)).astype(np.float32); a[:, 5] = np.where(g.random(500) < 0.9, -1, 1)
        pts.append(a)
    return infos, pts


def iou_boxes():
    g = np.random.default_rng(7)
    n = 300
    b = np.concatenate([g.uniform(-10, 10, (n, 3)), g.uniform(1, 5, (n, 3)), g.uniform(-3.2, 3.2, (n, 1))], 1).astype(np.float32)
    b[100:200, :2] = b[:100, :2] + g.normal(0, 0.2, (100, 2)).astype(np.float32)
    return b


def main(ref):
    src = open(os.path.join(ref, 'detection/detzero_det/datasets/dataset.py')).read()
    m = re.search(r'    @staticmethod\n    def merge_sweeps\(.*?\n        return point_clouds\n', src, re.S)
    ns = {'np': np}
    exec('class _T:\n' + m.group(0), ns)
    infos, pts = merge_sweeps_inputs()
    np.savez_compressed(os.path.join(HERE, 'merge_sweeps.npz'), want=ns['_T'].merge_sweeps(infos[0], infos, [p.copy() for p in pts]))

    import torch
    from oracle import build_ref
    build_ref.REF_SRC = os.path.join(ref, 'utils/detzero_utils/ops/iou3d_nms/src/iou3d_cpu.cpp')
    mod = build_ref.load() if os.path.exists(build_ref.SO) else (build_ref.build(), build_ref.load())[1]
    b = iou_boxes()
    out = torch.zeros(b.shape[0], b.shape[0])
    mod.boxes_iou_bev_cpu(torch.from_numpy(b), torch.from_numpy(b), out)
    np.savez_compressed(os.path.join(HERE, 'iou_bev.npz'), iou=out.numpy())


if __name__ == '__main__':
    main(sys.argv[1])

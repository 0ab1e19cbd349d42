"""oracle/refine_score_ref.py against the reference's golden vectors (tests/golden/refine_score.npz): the per-track targets, the
PRM / GRM / CRM recall records (keys, key order, values) and the CRM's IoU labels; and the C ABI the scoring adds."""
import os
import re

import numpy as np
import pytest

from detzero_b200 import _lib
from oracle import refine_score_ref as R
from oracle import track_gt_ref
from tests import refine_score_golden as G


def _scene():
    g, frames, tracks = G.load()
    assigned, _ = track_gt_ref.assign_track_target(frames, tracks, G.ASSIGN_THR)
    infos = R.attach_targets(assigned)
    return g, assigned, {tid: infos[tid] for tid in tracks}


def test_targets():
    g, assigned, infos = _scene()
    assert list(assigned['label']) == g['label_tk'].tolist() and list(assigned['unlabel']) == g['unlabel_tk'].tolist()
    assert [v['gt']['obj_ids'][0] for v in assigned['label'].values()] == g['label_obj'].tolist()
    assert [infos[t]['state'] == 'dynamic' for t in g['label_tk'].tolist()] == g['label_state'].tolist()
    assert infos[2]['matched'].tolist() == [True] * 20 + [False] * 5 and not infos[2]['gt_boxes_global'][20:].any()
    assert infos[6]['matched'].all() and not infos[6]['matched_tracklet'] and not infos[6]['gt_boxes_global'].any()
    assert infos[6]['state'] == 'dynamic' and infos[7]['state'] == 'static'        # the tracker's state on unmatched tracks
    assert [len(i['boxes_global']) for i in infos.values()] == [200, 25, 10, 10, 1, 10, 4]
    # a zero ground-truth box goes through the init-box transform like any other
    t = R.gt_pos_trajectory(infos[2])
    assert np.abs(t[:20, :2]).max() < 1.0 and np.abs(t[20:, :2]).max() > 1000.0


@pytest.mark.parametrize('centre', [False, True])
@pytest.mark.parametrize('cls', G.CLASS_NAMES)
def test_records(cls, centre):
    g, _, infos_all = _scene()
    rows = G.class_rows(g, cls)
    ids = g['tk_ids'].tolist()
    infos = {ids[b]: infos_all[ids[b]] for b in rows}
    th = G.THRESHOLDS[cls]
    world = [R.world_boxes(g['prm_pred'][b, :len(i['boxes_global'])], i['boxes_global'][len(i['boxes_global']) // 2])
             for b, i in zip(rows, infos.values())]
    prm, _, m1 = R.position_recall(infos, world, th, centre)
    grm, _, m2 = R.geometry_recall(infos, g['grm_pred'][rows], th, centre)
    assert min(m1['iou'].value, m2['iou'].value) > 1e-3, (m1['iou'].where, m2['iou'].where)
    for rec, model in ((prm, 'PRM'), (grm, 'GRM')):
        ref = G.record(g, model, cls)
        assert list(rec) == list(ref), model
        assert rec == ref, (model, {k: (rec[k], ref[k]) for k in rec if rec[k] != ref[k]})
    labels = R.refine_iou_labels(infos, world, g['grm_pred'][rows], centre)
    ref_labels = G.labels(g)
    for b, lab in zip(rows, labels):
        if centre:
            assert np.abs(lab - ref_labels[b]).max() < 2e-3            # the reference clips float32 world boxes 5 km out
        else:
            assert np.array_equal(lab, ref_labels[b])
    crm, m3 = R.confidence_recall(infos, [i['score'] for i in infos.values()],
                                  [g['crm_pred'][b, :len(i['boxes_global'])] for b, i in zip(rows, infos.values())],
                                  [ref_labels[b] for b in rows], th)
    ref = G.record(g, 'CRM', cls)
    assert list(crm) == g['CRM_%s_all_keys' % cls].tolist()
    assert {k: v for k, v in crm.items() if not isinstance(v, list)} == ref
    for k in ('gt_score', 'pred_score', 'ori_score'):
        assert np.array_equal(np.asarray(crm[k]), g['CRM_%s_%s' % (cls, k)]), k
    assert m3['score'].value > 0


def test_ratio_on_the_cut():
    """the pedestrian track's input ratio is exactly 0.7: counted by the PRM's >= and not by the GRM's >"""
    g, _, infos_all = _scene()
    assert G.record(g, 'PRM', 'Pedestrian')['Track level input (static) 0.5'] == 1
    assert G.record(g, 'GRM', 'Pedestrian')['Track level input (static) 0.5'] == 0
    _, _, m = R.geometry_recall({3: infos_all[3]}, g['grm_pred'][[2]], [0.5])
    assert m['ratio'].value < 1e-7


def test_c_abi_declares_the_scoring_entry_points():
    names = ('dz_refine_targets', 'dz_boxes_iou3d_aligned', 'dz_refine_score', 'dz_confidence_score')
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'detzero_b200.h')).read()
    for n in names:
        assert n in _lib.exported_symbols()
        m = re.search(r'\bint %s\(([^;]*)\);' % n, header)
        assert m, n
        assert len(m.group(1).split(',')) == len(_lib._SIGS[n][1]), n

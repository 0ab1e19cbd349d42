"""oracle/combine_ref.py (convert_frame_format + combine_det restated in numpy) against the reference's own combine_final
(tests/golden/combine.npz), exactly, for combine_conf_res on and off, with and without the dropped detections."""
import numpy as np
import pytest

from oracle import combine_ref
from tests import combine_golden as cg


@pytest.mark.parametrize('variant', list(cg.VARIANTS))
def test_oracle_vs_reference_golden(variant):
    g = cg.load()
    want = cg.expected(g, variant)
    combine_ref.assert_frames_equal(cg.oracle_frames(g, variant), want)
    conf, drop = cg.VARIANTS[variant]
    ids = [d['frame_id'] for d in want if d['sequence_name'] == 'seq_a']
    assert ids != sorted(ids)                                              # first-appearance order, not sorted
    n_drop = sum(len(d['score']) - len(d['obj_ids']) for d in want)
    assert (n_drop > 0) == drop


def test_golden_scene_covers_the_edge_cases():
    g = cg.load()
    want = {(d['sequence_name'], d['frame_id']): d for d in cg.expected(g, 'c1d1')}
    fid = g['s1_frame_ids']
    assert ('seq_b', int(fid[1])) not in want and g['s1_counts'][1] > 0 and not g['s1_kept'][1, :g['s1_counts'][1]].any()
    d = want[('seq_b', int(fid[4]))]
    assert len(d['score']) == len(d['obj_ids']) and g['s1_counts'][4] > 0     # an empty drop entry
    assert {tuple(sorted(set(d['name'][:len(d['obj_ids'])]))) for d in want.values()} >= {('Pedestrian', 'Vehicle')}
    n = np.concatenate([cg.tables(g, s)['box_num'] for s in (0, 1)])
    assert n.min() == 1 and n.max() == 200
    drops = np.concatenate([d['boxes_lidar'][len(d['obj_ids']):, 6] for d in want.values()])
    assert np.abs(g['s0_det'][..., 6]).max() > 2 * np.pi and np.all(np.abs(drops) <= np.float32(np.pi))


def test_missing_drop_entry_gives_no_dropped_row():
    g = cg.load()
    t = cg.tables(g, 1)
    drop = cg.det_drop(g, 1)
    key = str(int(t['frame_ids'][10]))
    assert len(drop[key]['score']) > 0
    del drop[key]
    out = combine_ref.frame_list(t['prm_lidar'], t['grm_pred'], t['crm'], t['frame_of_box'], t['box_num'], t['cls'], t['track_id'],
                                 t['poses'], 'seq_b', t['frame_ids'], drop)
    d = next(x for x in out if x['frame_id'] == int(key))
    assert len(d['score']) == len(d['obj_ids'])

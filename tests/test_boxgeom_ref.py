"""CPU check of the float64 box-geometry references in tests/boxgeom_ref.py against the oracle's float32 restatement of the
rotated-BEV overlap (oracle.c, the same algorithm as csrc/boxgeom.cuh).  The GPU tests trust these references and bounds; this
is what pins them without a GPU."""
import numpy as np
import pytest

import oracle
from tests import boxgeom_ref as gr

N = 400


def _oracle_overlap(a, b):
    return np.array([oracle.boxes_overlap_bev(a[i:i + 1], b[i:i + 1])[0, 0] for i in range(a.shape[0])], np.float64)


@pytest.mark.parametrize('family', gr.FAMILIES)
def test_oracle_overlap_inside_envelope_and_restatement(family):
    a, b = gr.pair_family(family, N)
    got = _oracle_overlap(a, b)
    lo, hi = gr.exact_overlap(a, b), gr.exact_overlap(a, b, gr.MARGIN)
    ref, margin = gr.restated_overlap(a, b)
    bound = gr.overlap_bound(a, b)
    assert np.all(got >= lo - bound), (family, (lo - bound - got).max())
    assert np.all(got <= hi + bound), (family, (got - hi - bound).max())
    sure = margin > 1
    assert np.all(np.abs(got - ref)[sure] <= bound[sure]), (family, (np.abs(got - ref) - bound)[sure].max())
    # the restatement itself lies in the envelope (no rounding to allow for beyond float64's)
    assert np.all(ref >= lo - 1e-9) and np.all(ref <= hi + 1e-9), family


def test_families_reach_the_edges_they_are_for():
    """the decision margin separates the degenerate families from the generic ones, and the envelope is wide where it should be"""
    frac = {f: np.mean(gr.restated_overlap(*gr.pair_family(f, N))[1] > 1) for f in gr.FAMILIES}
    assert frac['random'] > 0.9 and frac['near_duplicate'] > 0.5, frac
    assert frac['identical'] == 0 and frac['abutting'] < 0.1, frac
    a, b = gr.pair_family('rot_k_half_pi', N)
    sq = slice(0, N, 4)
    width = gr.exact_overlap(a[sq], b[sq], gr.MARGIN) - gr.exact_overlap(a[sq], b[sq])
    assert width.max() > 0.01, width.max()            # same-centre squares turned by k*pi/2: the margin adds a whole frame
    a, b = gr.pair_family('world_offset', N)
    assert np.all(gr.overlap_bound(a, b) > 1e-4) and np.all(np.abs(a[:, :2]).max(1) > 500)
    a, b = gr.pair_family('far_pair_edge', N)
    far = gr.far_pair(a, b)
    assert 0.2 < far.mean() < 0.8, far.mean()


def test_far_pair_means_no_overlap():
    """far_pair's promise, on the oracle: beyond the sum of the half-diagonals plus 0.05 m the overlap is exactly 0"""
    a, b = gr.pair_family('far_pair_edge', N)
    far = gr.far_pair(a, b)
    assert np.all(_oracle_overlap(a[far], b[far]) == 0)
    assert np.all(gr.exact_overlap(a[far], b[far], gr.MARGIN) == 0)


def test_exact_overlap_closed_forms():
    """the clip against hand-computed overlaps: axis-aligned offset boxes, a box inside another, a square turned by 45 degrees
    about a shared centre (area 8 * (sqrt(2) - 1) * h^2 for half-side h), and a grown pair"""
    a = np.array([[0, 0, 0, 4, 2, 1, 0], [0, 0, 0, 4, 4, 1, 0], [0, 0, 0, 2, 2, 1, 0], [0, 0, 0, 4, 2, 1, 0]], np.float32)
    b = np.array([[1, 0.5, 0, 4, 2, 1, 0], [0.5, 0, 0, 1, 1, 1, 0.3], [0, 0, 0, 2, 2, 1, np.pi / 4], [5, 0, 0, 4, 2, 1, 0]],
                 np.float32)
    want = [3 * 1.5, 1.0, 8 * (np.sqrt(2) - 1), 0.0]
    assert np.allclose(gr.exact_overlap(a, b), want, rtol=0, atol=1e-7)
    assert np.isclose(gr.exact_overlap(a[3:], b[3:], 0.5)[0], 0.0, atol=1e-12)       # gap 1 m, closed by 2 x 0.5 m
    assert np.isclose(gr.exact_overlap(a[3:], b[3:], 0.75)[0], 0.5 * 3.5, atol=1e-12)

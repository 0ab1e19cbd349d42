"""float64 references for the rotated-BEV box geometry of csrc/boxgeom.cuh (bev_overlap, bev_iou, iou3d, far_pair).

Two references, used together:

  * ``exact_overlap(a, b, infl)``: the area of the intersection of two rectangles, each grown by ``infl`` metres on every side,
    by convex polygon clipping in float64.  ``bev_overlap`` counts a corner as inside the other box when it lies within the
    1e-2 in-box margin of it, so its result is not the exact overlap but lies in the envelope
    [exact_overlap(a, b, 0), exact_overlap(a, b, MARGIN)]: every point it collects lies inside both boxes grown by the margin,
    and every vertex of the exact intersection is collected.
  * ``restated_overlap(a, b)``: bev_overlap's own algorithm (edge crossings with the strict sign test behind a bounding-box
    test, corners inside the other box by the margin, angular sort about the mean point, shoelace) in float64.  With it comes
    each pair's decision margin: how far the closest of those discrete tests is from flipping, in units of that test's own
    float32 rounding bound.  Where the margin exceeds 1 the float32 kernel took every decision the float64 restatement took,
    and the two results agree within ``overlap_bound``.

The bounds are derived from float32's unit roundoff U = 2^-24 and the largest coordinate of the pair, so they grow with the
distance of the boxes from the origin (the tracker associates boxes in world coordinates, kilometres from it).
"""
import numpy as np

U = 2.0 ** -24                                  # float32 unit roundoff
MARGIN = float(np.float32(1e-2))                # the in-box margin constant 1e-2f of inside_box
SX = np.array([-1.0, 1.0, 1.0, -1.0])           # corner order of box_corners: (-,-), (+,-), (+,+), (-,+), counter-clockwise
SY = np.array([-1.0, -1.0, 1.0, 1.0])


def _f64(boxes):
    return np.asarray(boxes, np.float32).astype(np.float64).reshape(-1, 7)


def corners(boxes, infl=0.0, origin=None):
    """(N, 7) boxes -> (N, 4, 2) float64 corners, each half-extent grown by `infl`, relative to `origin` (N, 2) if given (the
    difference of two float32 coordinates is exact in float64, so a clip near the origin keeps its precision kilometres away)"""
    b = _f64(boxes)
    hx, hy = b[:, 3:4] / 2 + infl, b[:, 4:5] / 2 + infl
    c, s = np.cos(b[:, 6:7]), np.sin(b[:, 6:7])
    lx, ly = SX * hx, SY * hy
    cx, cy = b[:, 0:1], b[:, 1:2]
    if origin is not None:
        cx, cy = cx - origin[:, 0:1], cy - origin[:, 1:2]
    return np.stack([cx + lx * c - ly * s, cy + lx * s + ly * c], axis=2)


def _clip_area(P, Q):
    """area of convex polygon P clipped by the counter-clockwise convex polygon Q (Sutherland-Hodgman)"""
    out = [p for p in P]
    for i in range(len(Q)):
        a, b = Q[i], Q[(i + 1) % len(Q)]
        inp, out = out, []
        if not inp:
            break
        side = [(b[0] - a[0]) * (p[1] - a[1]) - (b[1] - a[1]) * (p[0] - a[0]) for p in inp]
        for j in range(len(inp)):
            k = (j + 1) % len(inp)
            if side[j] >= 0:
                out.append(inp[j])
            if (side[j] >= 0) != (side[k] >= 0):
                t = side[j] / (side[j] - side[k])
                out.append(inp[j] + t * (inp[k] - inp[j]))
    if len(out) < 3:
        return 0.0
    P = np.array(out)
    return 0.5 * abs(np.dot(P[:, 0], np.roll(P[:, 1], -1)) - np.dot(P[:, 1], np.roll(P[:, 0], -1)))


def exact_overlap(a, b, infl=0.0):
    """(N, 7), (N, 7) -> (N,) exact BEV overlap area of row i with row i, both boxes grown by `infl` on every side"""
    o = _f64(a)[:, :2]
    A, B = corners(a, infl, o), corners(b, infl, o)
    return np.array([_clip_area(A[i], B[i]) for i in range(A.shape[0])])


def coord_error(a, b):
    """(N,) bound on the float32 error of any point bev_overlap collects, in metres; M = the largest |coordinate| of the pair,
    H = the larger hx + hy.  A corner (box_corners): x + sx*hx rounds by <= U*M, and subtracting x again carries that error into
    the offset (<= U*M + U*hx); cosf / sinf are off by <= 2 ulp <= 2U; the two products, their sum and + x round once each:
    <= (|cos| + |sin|) * U*M + U*M + 5U*H <= 3U*M + 5U*H.  A crossing point (s5*q0 - s1*q1) / (s5 - s1) with s1, s5 of opposite
    sign: two products, a difference and a division of terms bounded by |s5 - s1| * M add <= 4U*M (the error of s1 and s5
    slides it along its edges, which overlap_bound counts per unit of edge length)."""
    a, b = _f64(a), _f64(b)
    M = np.maximum(np.abs(a[:, :2]).max(1) + (a[:, 3] + a[:, 4]) / 2, np.abs(b[:, :2]).max(1) + (b[:, 3] + b[:, 4]) / 2)
    H = np.maximum(a[:, 3] + a[:, 4], b[:, 3] + b[:, 4]) / 2
    return 7 * U * M + 5 * U * H


def overlap_bound(a, b):
    """(N,) bound on |float32 bev_overlap - float64 restatement| when both took the same decisions, in m^2.
    Moving every vertex of the polygon by at most eps across the edges through it changes the area by at most eps times the
    perimeter of the polygon, which is at most min(Pa, Pb) grown by the margin (a convex set inside a convex box); a crossing
    point of two nearly parallel edges slides along them by eps / sin(angle), which changes the area by the same eps per unit of
    edge length.  The angular sort may swap two points
    whose angles differ by less than their rounding (eps / r); the swap changes the area by r * eps <= eps * D.  The shoelace
    sums at most 24 terms of at most D^2 (D = the larger inflated diagonal), each with 3 roundings plus the accumulation:
    <= 4 * 24 * U * D^2."""
    a, b = _f64(a), _f64(b)
    eps = coord_error(a, b)
    P = 2 * np.minimum(a[:, 3] + a[:, 4], b[:, 3] + b[:, 4]) + 8 * MARGIN
    D = np.maximum(np.hypot(a[:, 3], a[:, 4]), np.hypot(b[:, 3], b[:, 4])) + 4 * MARGIN
    return eps * (P + D) + 96 * U * D * D


def _cross_o(a, b, o):
    return (a[..., 0] - o[..., 0]) * (b[..., 1] - o[..., 1]) - (b[..., 0] - o[..., 0]) * (a[..., 1] - o[..., 1])


def _cross_err(a, b, o, eps):
    """float32 error bound of cross_o when every point carries eps: eps * (|a-o|_1 + |b-o|_1) from a and b, as much again from
    o, and 3 roundings of the products and their difference"""
    na, nb = np.abs(a - o).sum(-1), np.abs(b - o).sum(-1)
    return 2 * eps * (na + nb) + 3 * U * na * nb


def restated_overlap(a, b):
    """(N, 7), (N, 7) -> (area (N,), margin (N,)): bev_overlap's algorithm in float64 and the pair's decision margin, the
    smallest |signed margin| over the 16 edge-pair tests and the 8 in-box tests, each in units of its own rounding bound.
    An AND of tests flips as soon as its smallest signed margin does: its signed margin is their min (an OR: the max)."""
    a, b = _f64(a), _f64(b)
    n = a.shape[0]
    eps = coord_error(a, b)[:, None]
    A, B = corners(a), corners(b)
    A5, B5 = np.concatenate([A, A[:, :1]], 1), np.concatenate([B, B[:, :1]], 1)
    # ---- edge crossings: seg_hit(A[i+1], A[i], B[j+1], B[j]), i major
    p1, p0 = A5[:, 1:, None, :], A5[:, :-1, None, :]                # (n, 4, 1, 2)
    q1, q0 = B5[:, None, 1:, :], B5[:, None, :-1, :]                # (n, 1, 4, 2)
    p1, p0, q1, q0 = [np.broadcast_to(t, (n, 4, 4, 2)) for t in (p1, p0, q1, q0)]
    e = eps[:, :, None]
    bb = np.minimum.reduce([np.maximum(q0[..., d], q1[..., d]) - np.minimum(p0[..., d], p1[..., d]) for d in (0, 1)] +
                           [np.maximum(p0[..., d], p1[..., d]) - np.minimum(q0[..., d], q1[..., d]) for d in (0, 1)]) / (2 * e)
    s1, s2 = _cross_o(q0, p1, p0), _cross_o(p1, q1, p0)
    s3, s4 = _cross_o(p0, q1, q0), _cross_o(q1, p1, q0)
    n1, n2 = s1 / _cross_err(q0, p1, p0, e), s2 / _cross_err(p1, q1, p0, e)
    n3, n4 = s3 / _cross_err(p0, q1, q0, e), s4 / _cross_err(q1, p1, q0, e)
    same12 = np.maximum(np.minimum(n1, n2), np.minimum(-n1, -n2))   # s1 * s2 > 0
    same34 = np.maximum(np.minimum(n3, n4), np.minimum(-n3, -n4))
    seg = np.minimum(bb, np.minimum(same12, same34))                 # bb && s1*s2 > 0 && s3*s4 > 0
    hit = (bb >= 0) & (s1 * s2 > 0) & (s3 * s4 > 0)
    s5 = _cross_o(q1, p1, p0)
    with np.errstate(divide='ignore', invalid='ignore'):
        t = s5 - s1
        X = np.stack([(s5 * q0[..., 0] - s1 * q1[..., 0]) / t, (s5 * q0[..., 1] - s1 * q1[..., 1]) / t], -1)
    X = np.where(hit[..., None], X, 0.0)
    # ---- corners inside the other box by the margin: B[k] in a, then A[k] in b (the kernel's insertion order)
    def inside(box, P):
        d = P - box[:, None, :2]
        c, s = np.cos(-box[:, 6:7]), np.sin(-box[:, 6:7])
        rx, ry = d[..., 0] * c - d[..., 1] * s, d[..., 0] * s + d[..., 1] * c
        hx, hy = box[:, 3:4] / 2 + MARGIN, box[:, 4:5] / 2 + MARGIN
        err = 2 * eps + 8 * U * np.abs(d).sum(-1) + U * np.maximum(hx, hy)
        m = np.minimum(hx - np.abs(rx), hy - np.abs(ry)) / err
        return (np.abs(rx) < hx) & (np.abs(ry) < hy), m
    inB, mB = inside(a, B)
    inA, mA = inside(b, A)
    pts = np.concatenate([X.reshape(n, 16, 2), np.stack([B, A], 2).reshape(n, 8, 2)], 1)
    valid = np.concatenate([hit.reshape(n, 16), np.stack([inB, inA], 2).reshape(n, 8)], 1)
    margin = np.minimum(np.abs(seg).reshape(n, 16).min(1), np.minimum(np.abs(mB).min(1), np.abs(mA).min(1)))
    # ---- angular sort about the mean point, shoelace fan from the first point
    cnt = valid.sum(1)
    with np.errstate(invalid='ignore', divide='ignore'):
        cen = np.where(valid[..., None], pts, 0).sum(1) / cnt[:, None]
    ang = np.where(valid, np.arctan2(pts[..., 1] - cen[:, None, 1], pts[..., 0] - cen[:, None, 0]), np.inf)
    order = np.argsort(ang, axis=1, kind='stable')
    P = np.take_along_axis(pts, order[..., None], 1)
    ok = np.take_along_axis(valid, order, 1)
    d = P - P[:, :1]
    terms = d[:, :-1, 0] * d[:, 1:, 1] - d[:, :-1, 1] * d[:, 1:, 0]
    area = np.abs(np.where(ok[:, 1:], terms, 0).sum(1)) / 2
    area = np.where(cnt >= 3, area, 0.0)
    return area, margin


def iou_from_overlap(a, b, so):
    """bev_iou's formula on a given overlap"""
    a, b = _f64(a), _f64(b)
    return so / np.maximum(a[:, 3] * a[:, 4] + b[:, 3] * b[:, 4] - so, 1e-8)


def iou_bound(a, b, so, d_so):
    """bound on |bev_iou(float32) - iou_from_overlap(so)| when the float32 overlap is within d_so of so: the derivative of
    so / (S - so) in so is S / (S - so)^2; the areas, the subtraction and the division add 4 roundings relative to the IoU"""
    a, b = _f64(a), _f64(b)
    S = a[:, 3] * a[:, 4] + b[:, 3] * b[:, 4]
    un = np.maximum(S - so - d_so, 1e-8)
    return d_so * S / un ** 2 + 4 * U * so / un


def far_pair(a, b):
    """far_pair in float64: centre distance beyond the sum of the half-diagonals plus 0.05 m"""
    a, b = _f64(a), _f64(b)
    r = 0.5 * (np.hypot(a[:, 3], a[:, 4]) + np.hypot(b[:, 3], b[:, 4])) + 0.05
    return np.hypot(a[:, 0] - b[:, 0], a[:, 1] - b[:, 1]) > r


# ---- pair families: the degenerate configurations real detections and tracks produce -----------------------------------------
FAMILIES = ('random', 'near_duplicate', 'identical', 'rot_k_half_pi', 'abutting', 'nested', 'pedestrian', 'heading_wrap',
            'world_offset', 'zero_size', 'far_pair_edge')


def _base(g, n, size=(0.3, 5.0), span=40.0):
    return np.concatenate([g.uniform(-span, span, (n, 2)), g.uniform(-1, 1, (n, 1)), g.uniform(*size, (n, 2)),
                           g.uniform(1, 2, (n, 1)), g.uniform(-np.pi, np.pi, (n, 1))], 1)


def pair_family(name, n, seed=0):
    """(a, b) float32 (n, 7) pairs of one family"""
    g = np.random.default_rng([seed, FAMILIES.index(name)])
    a = _base(g, n)
    b = a.copy()
    if name == 'random':
        b = a.copy()
        b[:, :2] += g.uniform(-4, 4, (n, 2))
        b[:, 2:] = _base(g, n)[:, 2:]
    elif name == 'near_duplicate':
        b[:, :2] += g.normal(0, 0.3, (n, 2))
        b[:, 3:5] = np.maximum(b[:, 3:5] + g.normal(0, 0.05, (n, 2)), 0.2)
        b[:, 6] += g.normal(0, 0.05, n)
    elif name == 'identical':
        pass
    elif name == 'rot_k_half_pi':                       # collinear or perpendicular edges; a square with itself every 4th pair
        b[:, 6] += g.integers(1, 4, n) * (np.pi / 2)
        b[::4, 4] = b[::4, 3]
        a[::4, 4] = a[::4, 3]
        b[1::4, :2] += g.normal(0, 0.2, (len(b[1::4]), 2))
    elif name == 'abutting':                            # b shares a's front face, or lies along its side face (any length)
        c, s = np.cos(a[:, 6]), np.sin(a[:, 6])
        side = g.integers(0, 2, n).astype(bool)
        b[:, 3] = np.where(side, g.uniform(0.3, 5.0, n), b[:, 3])
        off = np.where(side, (a[:, 4] + b[:, 4]) / 2, (a[:, 3] + b[:, 3]) / 2)
        along = np.where(side, g.uniform(-1, 1, n), 0.0)
        b[:, 0] = a[:, 0] + np.where(side, -s, c) * off + c * along
        b[:, 1] = a[:, 1] + np.where(side, c, s) * off + s * along
    elif name == 'nested':                              # b strictly inside a, same or rotated heading
        b[:, 3:5] = a[:, 3:5] * g.uniform(0.2, 0.5, (n, 2))
        b[:, 6] += g.choice([0.0, 0.3, np.pi / 2], n)
        b[:, :2] += (a[:, 3:5].min(1, keepdims=True) * 0.1) * g.uniform(-1, 1, (n, 2))
    elif name == 'pedestrian':                          # 0.3 - 1 m boxes a pedestrian apart
        a = _base(g, n, size=(0.3, 1.0))
        b = a.copy()
        b[:, :2] += g.normal(0, 0.3, (n, 2))
        b[:, 3:5] = g.uniform(0.3, 1.0, (n, 2))
        b[:, 6] = g.uniform(-np.pi, np.pi, n)
    elif name == 'heading_wrap':                        # the same pair with b's heading moved by 2*pi*k
        b[:, :2] += g.normal(0, 0.5, (n, 2))
        b[:, 6] = g.uniform(-np.pi, np.pi, n)
        a[:, 6] += 2 * np.pi * g.integers(-3, 4, n)
        b[:, 6] += 2 * np.pi * g.integers(-3, 4, n)
    elif name == 'world_offset':                        # near-duplicates 1e3 - 1e4 m from the origin (world frame)
        b[:, :2] += g.normal(0, 0.3, (n, 2))
        b[:, 6] += g.normal(0, 0.05, n)
        off = g.uniform(1e3, 1e4, (n, 1)) * np.stack([np.cos(t := g.uniform(-np.pi, np.pi, n)), np.sin(t)], 1)
        a[:, :2] += off
        b[:, :2] += off
    elif name == 'zero_size':                           # a zero-length or zero-width box against a normal one, and two of them
        k = g.integers(0, 2, n)
        a[np.arange(n), 3 + k] = 0.0
        b[:, :2] += g.normal(0, 0.5, (n, 2))
        b[:, 6] = g.uniform(-np.pi, np.pi, n)
        both = np.arange(n) % 3 == 0
        b[both, 3 + k[both]] = 0.0
    elif name == 'far_pair_edge':                       # centre distance at the far_pair radius, either side of it
        b[:, 3:5] = g.uniform(0.3, 5.0, (n, 2))
        b[:, 6] = g.uniform(-np.pi, np.pi, n)
        r = 0.5 * (np.hypot(a[:, 3], a[:, 4]) + np.hypot(b[:, 3], b[:, 4])) + 0.05
        t = g.uniform(-np.pi, np.pi, n)
        dist = r * (1 + g.choice([-1e-3, -1e-5, 1e-5, 1e-3, 0.05], n))
        b[:, 0], b[:, 1] = a[:, 0] + dist * np.cos(t), a[:, 1] + dist * np.sin(t)
    else:
        raise KeyError(name)
    return a.astype(np.float32), b.astype(np.float32)

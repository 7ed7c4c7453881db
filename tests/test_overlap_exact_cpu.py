"""Box-footprint overlaps against exact rational arithmetic (oracle/exact_overlap.py), on the CPU.

The NMS and evaluator oracles (oracle.postprocess, oracle.kitti_eval) are what every GPU test of pg_postprocess,
pg_nms_boxes_3d and pg_kitti_eval trusts, and they share their Sutherland-Hodgman clipper with the kernels.  Here
they are checked against an exact intersection computed by a different algorithm, on hand-derived cases, random pairs
and box pairs aimed at the NMS (0.01, 0.5) and KITTI (0.5, 0.7) thresholds.  The boundary-family generator lives here
and is reused by tests/test_overlap_exact_gpu.py."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import exact_overlap as ex
from oracle import kitti_eval as ke
from oracle import postprocess as pp

NMS_THRESHOLDS = (0.01, 0.5)
KITTI_THRESHOLDS = (0.5, 0.7)
DELTAS = (1e-3, 1e-6, 1e-9)
FAMILIES = ('yaw0', 'equal_yaw', 'perpendicular', 'general', 'near_parallel', 'containment', 'shared_edge', 'thin',
            'far', 'height_shift', 'height_nested')


def _rect(x0, z0, x1, z1):
    return np.array([[x1, z1], [x1, z0], [x0, z0], [x0, z1]], np.float64)


# ---------------------------------------------------------------------------------------------
# boundary families: box pairs (x, y, z, l, h, w, yaw) whose overlap is aimed at t (1 +- delta)
# ---------------------------------------------------------------------------------------------
def _variant(rng, family):
    """Random base parameters of one family member."""
    v = dict(x=rng.uniform(-20, 20), y=rng.uniform(0.5, 2.0), z=rng.uniform(5, 50), l=rng.uniform(1.0, 5.0),
             w=rng.uniform(0.5, 2.0), h=rng.uniform(1.0, 2.0), yaw=rng.uniform(-np.pi, np.pi),
             dir=rng.uniform(-np.pi, np.pi), dyaw=rng.uniform(0.2, 1.3))
    if family in ('yaw0', 'shared_edge'):
        v.update(x=float(rng.integers(-64, 64)) / 4, z=float(rng.integers(20, 200)) / 4, y=1.0,
                 l=float(rng.choice([2.0, 4.0])), w=float(rng.choice([1.0, 2.0])), h=float(rng.choice([1.0, 2.0])),
                 yaw=0.0)
    if family == 'yaw0':
        v['dir'] = float(rng.choice([0.0, np.pi / 2])) if rng.random() < 0.5 else v['dir']
    if family == 'thin':
        v['w'] = 1e-3 * v['l']
    if family == 'far':
        v.update(x=rng.choice([-1, 1]) * rng.uniform(900, 1100), z=rng.choice([-1, 1]) * rng.uniform(900, 1100))
    return v


def family_pair(family, s, v):
    """-> (a, b) float64 boxes for shift / size parameter s; the overlap decreases as s grows over family_range."""
    x, y, z, l, h, w, yaw = v['x'], v['y'], v['z'], v['l'], v['h'], v['w'], v['yaw']
    a = [x, y, z, l, h, w, yaw]
    dx, dz = math.cos(v['dir']), math.sin(v['dir'])
    if family in ('yaw0', 'equal_yaw', 'perpendicular', 'general', 'near_parallel', 'far'):
        yb = {'perpendicular': yaw + np.pi / 2, 'general': yaw + v['dyaw'], 'near_parallel': yaw + 1e-6}.get(family, yaw)
        if family == 'far':
            yb = yaw + v['dyaw']
        b = [x + s * dx, y, z + s * dz, l, h, w, yb]
    elif family == 'containment':      # a inside b: b longer by the factor s
        b = [x, y + 0.05 * h, z, l * s, 1.1 * h, 1.2 * w, yaw]
    elif family == 'shared_edge':      # b: 3/4 as wide, one long edge on a's; slides along it
        b = [x + s, y, z + w / 8, l, h, 0.75 * w, yaw]
    elif family == 'thin':             # slides along the long axis
        b = [x + s * math.cos(yaw), y, z - s * math.sin(yaw), l, h, w, yaw]
    elif family == 'height_shift':
        b = [x, y - s, z, l, h, w, yaw]
    elif family == 'height_nested':    # b's height range nested in a's, shrinking
        b = [x, y - s * h / 2, z, l, h * (1 - s), w, yaw]
    else:
        raise ValueError(family)
    return np.array(a), np.array(b)


def family_range(family, v):
    return {'containment': (1.0, 200.0), 'shared_edge': (0.0, v['l']),
            'height_shift': (0.0, v['h']), 'height_nested': (0.0, 1.0)}.get(family, (0.0, v['l'] + v['w']))


def nms_fast_iou(a, b):
    """The float64 NMS oracle on float32 boxes (a = single box)."""
    c = pp.boxes_3d_to_corners(np.stack([a, b]).astype(np.float32))
    return float(pp.overlapped_boxes_3d_fast_poly(c[0], c[1:])[0])


def kitti_rows(a, b, alpha=0.0, score=0.5):
    """Ground-truth and detection rows [14] / [15] of boxes a (ground truth) and b (detection), 2-D boxes equal."""
    def geo(box):
        x, y, z, l, h, w, yaw = (float(v) for v in box)
        return [h, w, l, x, y, z, yaw]
    img = [100.0, 100.0, 300.0, 200.0]
    g = np.array([0.0, 0.0, alpha] + img + geo(a))
    d = np.array([-1.0, -1.0, alpha] + img + geo(b) + [score])
    return g, d


def kitti_fast_overlap(a, b, metric, criterion=-1):
    g, d = kitti_rows(a, b)
    return float(ke.overlaps(g[None], [5 if criterion == 0 else 0], d[None])[metric, 0, 0])


def _aim(fn, lo, hi, target, steps):
    """Bisection on a decreasing fn: (s_above, s_below) with fn(s_above) >= target > fn(s_below)."""
    for _ in range(steps):
        mid = 0.5 * (lo + hi)
        if mid in (lo, hi):
            break
        if fn(mid) >= target:
            lo = mid
        else:
            hi = mid
    return lo, hi


def _reachable(rng, family, fn, target, tries=50):
    """A family member whose overlap falls from above target to below it over its parameter range."""
    for _ in range(tries):
        v = _variant(rng, family)
        lo, hi = family_range(family, v)
        top, bottom = fn(lo, v), fn(hi, v)
        if top >= target > bottom:
            return v, lo, hi
    raise RuntimeError('%s never reaches %g' % (family, target))


def nms_families(variants=1, seed=0, families=FAMILIES, thresholds=NMS_THRESHOLDS, deltas=DELTAS):
    """-> list of dict(family, t, delta, side, a, b): float32 boxes aimed at IoU t (1 + side * delta)."""
    rng = np.random.default_rng(seed)
    out = []
    for fam in families:
        for t in thresholds:
            for delta in deltas:
                for side in (1, -1):
                    for _ in range(variants):
                        fn = lambda s, v: nms_fast_iou(*family_pair(fam, s, v))   # noqa: E731
                        v, lo, hi = _reachable(rng, fam, fn, t * (1 + delta))
                        # 34 halvings take the shift below the float32 resolution of the boxes
                        above, below = _aim(lambda s: fn(s, v), lo, hi, t * (1 + side * delta), 34)
                        a, b = family_pair(fam, above if side > 0 else below, v)
                        out.append(dict(family=fam, t=t, delta=delta, side=side, a=a.astype(np.float32),
                                        b=b.astype(np.float32)))
    return out


def kitti_families(variants=1, seed=0, families=FAMILIES, thresholds=KITTI_THRESHOLDS, deltas=DELTAS, metric=1,
                   criterion=-1):
    """-> list of dict(family, t, delta, side, metric, criterion, gt [14], det [15]) aimed at overlap t (1 +- delta)."""
    rng = np.random.default_rng(seed)
    out = []
    for fam in families:
        if metric == 1 and fam.startswith('height') or criterion == 0 and fam == 'height_nested':
            continue                      # no height in the ground overlap; a nested detection is covered throughout
        for t in thresholds:
            for delta in deltas:
                for side in (1, -1):
                    for _ in range(variants):
                        fn = lambda s, v: kitti_fast_overlap(*family_pair(fam, s, v), metric, criterion)   # noqa: E731
                        v, lo, hi = _reachable(rng, fam, fn, t * (1 + delta))
                        # 48 halvings: the overlap within ~1e-13 of the aim, far inside delta
                        above, below = _aim(lambda s: fn(s, v), lo, hi, t * (1 + side * delta), 48)
                        g, d = kitti_rows(*family_pair(fam, above if side > 0 else below, v))
                        out.append(dict(family=fam, t=t, delta=delta, side=side, metric=metric, criterion=criterion,
                                        gt=g, det=d))
    return out


# ---------------------------------------------------------------------------------------------
# degenerate NMS cases: what the reference's nms.py does, one rule each
# ---------------------------------------------------------------------------------------------
def _box(x, z, l, h, w, yaw=0.0, y=1.0):
    return [x, y, z, l, h, w, yaw]


# (name, thres, boxes [first = higher score], kept by the merge / rescore variants, kept by the plain (int corner) one,
#  rule).  Both boxes have the same class.
DEGENERATE = [
    ('zero_length', 0.01, [_box(0, 10, 4, 1.5, 2), _box(0, 10, 0, 1.5, 2)], [0, 1], [0, 1],
     'a footprint of area 0 shares area 0: the IoU is 0, which does not exceed the threshold'),
    ('zero_width_rotated', 0.01, [_box(0, 10, 4, 1.5, 2, 0.3), _box(0.5, 10, 3, 1.5, 0, 0.3)], [0, 1], [0, 1],
     'the same for a rotated box of width 0'),
    ('zero_height_one', 0.01, [_box(0, 10, 4, 1.5, 2), _box(0.5, 10, 4, 0, 2, y=0.5)], [0, 1], [0, 1],
     'one box of height 0 inside the other\'s height range: shared_y 0, the IoU is 0'),
    ('zero_height_both', 0.01, [_box(0, 10, 4, 0, 2), _box(0.5, 10, 4, 0, 2)], [0, 1], [0],
     'both heights 0: the union is 0 and the IoU 0 / 0 = NaN; `NaN > thres` is false (kept) but bboxes_nms keeps only '
     'if `NaN <= thres`, which is false (removed)'),
    ('zero_length_both', 0.01, [_box(0, 10, 0, 1.5, 2), _box(0, 10, 0, 1.5, 2)], [0, 1], [0],
     'both footprints of area 0 and overlapping bounding boxes: NaN, as above'),
    ('touching_edge_thres0', 0.0, [_box(0, 10, 4, 1.5, 2), _box(4, 10, 4, 1.5, 2)], [0, 1], [0, 1],
     'boxes sharing an edge pass the early-out but share area 0: IoU 0, not > 0'),
    ('touching_vertex_thres0', 0.0, [_box(0, 10, 4, 1.5, 2), _box(4, 12, 4, 1.5, 2)], [0, 1], [0, 1],
     'boxes touching at a vertex: IoU 0'),
    ('touching_height_thres0', 0.0, [_box(0, 10, 4, 1.5, 2), _box(1, 10, 4, 1.5, 2, y=-0.5)], [0, 1], [0, 1],
     'height ranges touching: shared_y 0, IoU 0'),
    ('overlap_thres0', 0.0, [_box(0, 10, 4, 1.5, 2), _box(3.75, 10, 4, 1.5, 2)], [0], [0],
     'any positive overlap exceeds 0'),
    ('zero_length_inside_thres0', 0.0, [_box(0.3, 10.1, 4, 1.5, 2, 0.3), _box(0.1, 10.2, 0, 1.5, 2)], [0, 1], [0, 1],
     'thres 0: a footprint of area 0 inside the other still shares exactly 0 (the clip is skipped, not rounded)'),
    ('zero_length_inside_thres0_b', 0.0, [_box(-0.7, 9.3, 3, 1.5, 2.5, -1.1), _box(-0.45, 9.1, 0, 1.5, 1.3)], [0, 1],
     [0, 1], 'the same, another rotation'),
    ('zero_width_inside_thres0', 0.0, [_box(0.2, 10.3, 4, 1.5, 2, 2.2), _box(0.15, 10.05, 1.7, 1.5, 0)], [0, 1], [0, 1],
     'the same for a width of 0'),
    ('apart_zero_height_both', 0.01, [_box(0, 10, 4, 0, 2), _box(8, 10, 4, 0, 2)], [0, 1], [0, 1],
     'bounding boxes apart: the early-out gives 0 before any 0 / 0'),
]


# ---------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('a, b, want', [
    (_rect(0, 0, 2, 2), _rect(3, 0, 5, 2), 0),                 # disjoint
    (_rect(0, 0, 2, 2), _rect(2, 0, 4, 2), 0),                 # shared edge
    (_rect(0, 0, 2, 2), _rect(2, 2, 4, 4), 0),                 # shared vertex
    (_rect(0, 0, 2, 1), _rect(0, 0, 2, 1), 2),                 # identical
    (_rect(0, 0, 4, 4), _rect(1, 1, 2, 3), 2),                 # containment
    (_rect(0, 0, 4, 2), _rect(2, 0, 6, 2), 4),                 # half-overlapping rectangles
    (_rect(-1, -1, 1, 1), np.array([[1, 0], [0, 1], [-1, 0], [0, -1]], float), 2),      # diamond in a square
    (_rect(0, 0, 1, 1), np.array([[1, 0], [0, 1], [-1, 0], [0, -1]], float), Fraction(1, 2)),
    (_rect(0, 0, 2, 2), _rect(1, -1, 3, 1), 1),
    (_rect(0, 0, 0, 2), _rect(-1, -1, 1, 3), 0),               # zero-width quad
    (_rect(0, 0, 0, 0), _rect(-1, -1, 1, 3), 0),               # a point
])
def test_intersection_area_hand_cases(a, b, want):
    assert ex.intersection_area(a, b) == want
    assert ex.intersection_area(b, a) == want
    assert ex.intersection_area(a[::-1], b) == want           # orientation does not matter


def test_nms_iou_hand_cases():
    def iou(a, b):
        return ex.nms_iou(ex.nms_corners(a), ex.nms_corners(b))
    box = _box(1, 10, 4, 2, 2)
    assert iou(box, box) == 1.0
    assert iou(box, _box(3, 10, 4, 2, 2)) == 4 * 2 / (32 - 8)                     # half-overlapping: 1/3
    assert iou(box, _box(1, 10, 2, 2, 1)) == 4 / (16 + 4 - 4)                     # inside: 1/4
    assert iou(box, _box(5, 10, 4, 2, 2)) == 0.0                                  # shared edge
    assert iou(box, _box(5, 12, 4, 2, 2)) == 0.0                                  # shared vertex
    assert iou(box, _box(9, 10, 4, 2, 2)) == 0.0                                  # apart
    # 90 degrees: a 4 x 2 footprint against its rotation about the same centre shares 2 x 2
    rot = ex.nms_iou_interval(np.float32(box), np.float32(_box(1, 10, 4, 2, 2, np.pi / 2)))
    assert rot[0] <= 8 / 24 <= rot[1] and rot[1] - rot[0] < 2e-5
    # yaw +-pi: the same footprint, up to the float32 trig
    for yaw in (np.pi, -np.pi):
        lo, hi = ex.nms_iou_interval(np.float32(box), np.float32(_box(1, 10, 4, 2, 2, yaw)))
        assert lo <= 1.0 <= hi and hi - lo < 1e-4


def test_kitti_overlap_hand_cases():
    g, d = kitti_rows(_box(0, 10, 4, 2, 2), _box(2, 10, 4, 2, 2))
    assert ex.ground_overlap(g, d) == 4 / 12
    assert ex.ground_overlap(g, d, 0) == 0.5
    assert ex.box3d_overlap(g, d) == 8 / 24
    d2 = d.copy()
    d2[11] -= 1.0                         # height ranges overlap by half
    assert ex.box3d_overlap(g, d2) == 4 / (32 - 4)
    d2[11] -= 1.0                         # touching
    assert ex.box3d_overlap(g, d2) == 0.0
    d2[11] -= 1.0                         # disjoint: max(0, ...)
    assert ex.box3d_overlap(g, d2) == 0.0
    gi, di = g.copy(), d.copy()
    gi[3:7], di[3:7] = (100, 100, 200, 200), (150, 100, 250, 200)
    assert ex.image_overlap(di, gi) == 5000 / 15000
    assert ex.image_overlap(di, gi, 0) == 0.5
    di[3:7] = (200, 100, 300, 200)
    assert ex.image_overlap(di, gi) == 0.0


def test_invariants_on_random_pairs():
    rng = np.random.default_rng(1)
    for _ in range(60):
        a = ex.eval_footprint(rng.uniform(0.1, 5), rng.uniform(0.1, 3), rng.uniform(-2, 2), rng.uniform(-2, 2),
                              rng.uniform(-np.pi, np.pi))
        b = ex.eval_footprint(rng.uniform(0.1, 5), rng.uniform(0.1, 3), rng.uniform(-2, 2), rng.uniform(-2, 2),
                              rng.uniform(-np.pi, np.pi))
        ab = ex.intersection_area(a, b)
        assert ab == ex.intersection_area(b, a)
        assert ex.intersection_area(a, a) == ex.area(a)
        assert 0 <= ab <= min(ex.area(a), ex.area(b))


def _close(got, want, pts, shared):
    """Within 1e-12 relative, or within the fp64 rounding a clipper can make on coordinates of magnitude R when the
    shared area is small against R^2 (thin boxes, boxes far from the origin)."""
    if want == 0:
        return abs(got) <= 1e-14
    r = float(np.abs(pts).max())
    tol = max(1e-12, 16 * 2.0 ** -53 * r * r / float(shared)) if shared > 0 else 1e-12
    return abs(got - want) <= tol * abs(want)


_CACHE = {}


def default_nms_families():
    if 'nms' not in _CACHE:
        _CACHE['nms'] = nms_families()
    return _CACHE['nms']


def test_nms_oracle_matches_exact():
    rng = np.random.default_rng(2)
    pairs = [(p['a'], p['b']) for p in default_nms_families()]
    for _ in range(150):
        a = np.r_[rng.uniform(-5, 5), rng.uniform(0, 2), rng.uniform(5, 15), rng.uniform(0.5, 5, 3),
                  rng.uniform(-np.pi, np.pi)]
        b = a + np.r_[rng.normal(0, 1, 3), rng.normal(0, 0.3, 3), rng.normal(0, 1)]
        b[3:6] = np.abs(b[3:6])
        pairs.append((a.astype(np.float32), b.astype(np.float32)))
    hit = 0
    for a, b in pairs:
        c = pp.boxes_3d_to_corners(np.stack([a, b]))
        want = ex.nms_iou(c[0], c[1])
        got = pp.overlapped_boxes_3d_fast_poly(c[0], c[1:])[0]
        shared = ex.intersection_area(c[0][:4, [0, 2]], c[1][:4, [0, 2]])
        assert _close(got, want, c[:, :4, [0, 2]], shared), (a, b, got, want)
        hit += want > 0
    assert hit > 200


@pytest.mark.parametrize('metric', [1, 2])
def test_kitti_oracle_matches_exact(metric):
    fams = kitti_families(metric=metric) + kitti_families(metric=metric, criterion=0, thresholds=(0.7,),
                                                          deltas=(1e-6,), seed=5)
    assert len(fams) > 40
    for p in fams:
        g, d = p['gt'], p['det']
        want = (ex.ground_overlap if metric == 1 else ex.box3d_overlap)(g, d, p['criterion'])
        got = ke.overlaps(g[None], [5 if p['criterion'] == 0 else 0], d[None])[metric, 0, 0]
        gp, dp = ex.eval_footprint(*ex._row_fp(g)), ex.eval_footprint(*ex._row_fp(d))
        assert _close(got, want, np.stack([gp, dp]), ex.intersection_area(gp, dp)), (p['family'], got, want)
        got_img = ke.overlaps(g[None], [0], d[None])[0, 0, 0]
        assert got_img == ex.image_overlap(d, g) == 1.0


def test_families_land_on_both_sides_of_the_thresholds():
    """Every family is aimed at every threshold: the certified IoUs straddle it, closer as delta shrinks."""
    fams = default_nms_families()
    for fam in FAMILIES:
        mine = [p for p in fams if p['family'] == fam]
        assert mine, fam
        for t in NMS_THRESHOLDS:
            errs = [ex.nms_iou(ex.nms_corners(p['a']), ex.nms_corners(p['b'])) / t - 1 for p in mine if p['t'] == t]
            assert min(errs) < 0 < max(errs), (fam, t)
            assert min(abs(e) for e in errs) < 2e-3, (fam, t)


def test_intervals_contain_the_nominal_value():
    for p in nms_families(families=('general', 'near_parallel', 'thin', 'far'), deltas=(1e-3,)):
        v = ex.nms_iou(ex.nms_corners(p['a']), ex.nms_corners(p['b']))
        lo, hi = ex.nms_iou_interval(p['a'], p['b'])
        assert lo <= v <= hi and hi - lo < (5e-3 if p['family'] == 'thin' else 1e-3) * v, p['family']
        ilo, ihi = ex.nms_iou_interval(p['a'], p['b'], appr=100.0)
        assert not ilo > ihi


@pytest.mark.parametrize('case', DEGENERATE, ids=[c[0] for c in DEGENERATE])
def test_degenerate_rules_are_the_reference_nms(case):
    """The rule stated for each degenerate case is what the reference's own nms.py gives (needs the reference tree)."""
    try:
        _, nms = pp.reference_modules()
    except RuntimeError as e:
        pytest.skip(str(e))
    name, thres, boxes, keep_unc, keep_plain, _ = case
    boxes = np.array(boxes, np.float32)
    labels, scores = np.array([1, 1]), np.array([0.9, 0.5], np.float32)
    with np.errstate(invalid='ignore', divide='ignore'):
        out = nms.nms_boxes_3d_uncertainty(labels.copy(), boxes.copy(), scores.copy(), overlapped_thres=thres,
                                           overlapped_fn=nms.overlapped_boxes_3d_fast_poly, appr_factor=100.0,
                                           top_k=-1, attributes=np.arange(2))
        assert list(out[3]) == keep_unc
        out = nms.nms_boxes_3d(labels.copy(), boxes.copy(), scores.copy(), overlapped_thres=thres,
                               overlapped_fn=nms.overlapped_boxes_3d_fast_poly, appr_factor=100.0, top_k=-1,
                               attributes=np.arange(2))
        assert list(out[3]) == keep_plain


def test_degenerate_rules_follow_from_the_exact_overlap():
    """The same decisions from the exact formula: NaN never removes under `>`, always under `not <=`."""
    for name, thres, boxes, keep_unc, keep_plain, _ in DEGENERATE:
        a, b = np.array(boxes, np.float32)
        for appr, want, removes in ((None, keep_unc, lambda o: o > thres), (100.0, keep_plain,
                                                                             lambda o: not o <= thres)):
            ca, cb = ex.nms_corners(a, appr=appr), ex.nms_corners(b, appr=appr)
            ov = ex.nms_iou(ca, cb)
            assert ([0] if removes(ov) else [0, 1]) == want, (name, appr, ov)

"""Exact box-footprint overlaps in rational arithmetic: the independent check of the four fp64 clippers
(pg_geom.cuh's clipped_area, oracle.postprocess.clip_convex, oracle.kitti_eval and the Boost stand-in).

TEST INFRASTRUCTURE ONLY.  The float64 corners are taken exactly as each caller forms them and converted to
``fractions.Fraction``; from there everything is exact until the one float rounding the caller makes at its last
step.  The intersection of two convex quads is NOT computed by clipping: it is the convex polygon spanned by the
vertices of either quad that lie inside or on the other and by every edge-edge intersection point, ordered by angle
around an interior point (exact cross products) and measured with the shoelace formula.

Overlap formulas:

* ``nms_iou``: nms.py:64-88 (overlapped_boxes_3d_fast_poly): the bounding-box early-out, ``shared_y * shared_area``,
  ``np.float32(intersection) / (union - intersection)``; NaN where the union is zero.
* ``ground_overlap`` / ``box3d_overlap`` / ``image_overlap``: groundBoxOverlap, box3DOverlap and imageBoxOverlap of
  the reference evaluator (criterion -1: union, 0: detection area); the double quotient is the exact quotient rounded.

Perturbation intervals (``nms_iou_interval``, ``eval_overlap_interval``): the NMS kernel evaluates cos / sin with CUDA's
``cosf`` / ``sinf``, NumPy with its own float32 routine, the evaluator with CUDA's and glibc's double routines; each is
within a few ulp of the true value, so the corners legitimately differ in their last bits.  The interval encloses
every overlap over corners whose cos / sin are moved by up to ``k`` ulp, plus the fp64 rounding of the clippers
themselves (unless the caller states the configuration is computed exactly).  A decision against a threshold is only
certain when the whole interval lies on one side.
"""
import functools
import math
from fractions import Fraction

import numpy as np

TRIG_ULPS = 4          # |CUDA - NumPy / glibc| <= 2 + 2 ulp
_U = 2.0 ** -53


# ---------------------------------------------------------------------------------------------
# exact convex-quad geometry
# ---------------------------------------------------------------------------------------------
def _frac_pts(pts):
    return [(Fraction(float(x)), Fraction(float(z))) for x, z in np.asarray(pts, np.float64).reshape(-1, 2)]


def _cross(o, a, b):
    return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])


def _signed_area2(p):
    return sum(p[i][0] * p[(i + 1) % len(p)][1] - p[i][1] * p[(i + 1) % len(p)][0] for i in range(len(p)))


def area(pts):
    """|area| of a quad (float64 corners [4, 2]) as a Fraction."""
    return abs(_signed_area2(_frac_pts(pts))) / 2


def _inside(p, ccw):
    n = len(ccw)
    return all(_cross(ccw[i], ccw[(i + 1) % n], p) >= 0 for i in range(n))


def _seg_hits(p0, p1, q0, q1):
    """Intersection point of two non-parallel closed segments, or None (parallel overlaps add only endpoints,
    which the inside tests already collect)."""
    r = (p1[0] - p0[0], p1[1] - p0[1])
    s = (q1[0] - q0[0], q1[1] - q0[1])
    den = r[0] * s[1] - r[1] * s[0]
    if den == 0:
        return None
    w = (q0[0] - p0[0], q0[1] - p0[1])
    t = (w[0] * s[1] - w[1] * s[0]) / den
    u = (w[0] * r[1] - w[1] * r[0]) / den
    if 0 <= t <= 1 and 0 <= u <= 1:
        return (p0[0] + t * r[0], p0[1] + t * r[1])
    return None


def intersection_area(a, b):
    """Exact area of the intersection of two convex quads (float64 corners [4, 2], either orientation) -> Fraction.
    A quad of zero area gives exactly 0."""
    pa, pb = _frac_pts(a), _frac_pts(b)
    sa, sb = _signed_area2(pa), _signed_area2(pb)
    if sa == 0 or sb == 0:
        return Fraction(0)
    if sa < 0:
        pa = pa[::-1]
    if sb < 0:
        pb = pb[::-1]
    pts = {p for p in pa if _inside(p, pb)} | {p for p in pb if _inside(p, pa)}
    for i in range(4):
        for j in range(4):
            hit = _seg_hits(pa[i], pa[(i + 1) % 4], pb[j], pb[(j + 1) % 4])
            if hit is not None:
                pts.add(hit)
    if len(pts) < 3:
        return Fraction(0)
    pts = list(pts)
    n = len(pts)
    c = (sum(p[0] for p in pts) / n, sum(p[1] for p in pts) / n)

    def half(p):
        dx, dz = p[0] - c[0], p[1] - c[1]
        return 0 if (dz > 0 or (dz == 0 and dx > 0)) else 1

    def cmp(p, q):
        hp, hq = half(p), half(q)
        if hp != hq:
            return hp - hq
        x = _cross(c, p, q)
        return -1 if x > 0 else (1 if x < 0 else 0)

    pts.sort(key=functools.cmp_to_key(cmp))
    return abs(_signed_area2(pts)) / 2


def _quotient(num, den):
    """num / den rounded to float64 (den == 0: NaN for 0/0, else a signed infinity)."""
    if den == 0:
        return math.nan if num == 0 else math.copysign(math.inf, num)
    return float(Fraction(num) / den)


# ---------------------------------------------------------------------------------------------
# NMS: nms.py:9-27 corners and nms.py:64-88 overlap
# ---------------------------------------------------------------------------------------------
def nms_trig(yaw):
    """(cos, sin) as nms.py evaluates them for a float32 yaw: NumPy's float32 routines."""
    y = np.float32(yaw)
    return float(np.cos(y)), float(np.sin(y))


def nms_corners(box, trig=None, appr=None):
    """nms.py:9-27 for one float32 box [7] -> [8, 3] float64 corners: the half extents in float32, trig in float32
    (``trig`` overrides it), the rest in float64.  appr: np.int32(corners * appr) (bboxes_nms, nms.py:114)."""
    x, y, z, l, h, w, yaw = (np.float32(v) for v in box)
    c, s = nms_trig(yaw) if trig is None else trig
    hl, hw, hh = float(l / np.float32(2)), float(w / np.float32(2)), float(h)
    lx, lz = [hl, hl, -hl, -hl], [hw, -hw, -hw, hw]
    out = np.zeros((8, 3))
    for i in range(4):
        fx = (lx[i] * c + 0.0) + lz[i] * s + float(x)
        fz = (lx[i] * -s + 0.0) + lz[i] * c + float(z)
        out[i] = out[i + 4] = (fx, 0.0, fz)
    out[:4, 1] = 0.0 + float(y)
    out[4:, 1] = -hh + float(y)
    if appr is not None:
        out = np.int32(out * appr).astype(np.float64)
    return out


def _nms_parts(ca, cb):
    """Exact (inter, union) of nms.py:64-88 for two [8, 3] corner arrays, or None where the bounding boxes are
    apart (the early-out that returns 0)."""
    mx0, mn0, mx, mn = ca.max(0), ca.min(0), cb.max(0), cb.min(0)
    if np.any((mx0 < mn) | (mn0 > mx)):
        return None
    area1, area2 = area(ca[:4, [0, 2]]), area(cb[:4, [0, 2]])
    shared = intersection_area(ca[:4, [0, 2]], cb[:4, [0, 2]])
    f = Fraction
    shared_y = min(f(mx[1]), f(mx0[1])) - max(f(mn[1]), f(mn0[1]))
    inter = shared_y * shared
    union = (f(mx[1]) - f(mn[1])) * area2 + (f(mx0[1]) - f(mn0[1])) * area1
    return inter, union


def _f32_of(inter):
    """np.float32(intersection): the exact value rounded to float64 (the reference's variable), then to float32."""
    return Fraction(float(np.float32(float(inter))))


def nms_iou(ca, cb):
    """nms.py:64-88 of single box ``ca`` against ``cb`` ([8, 3] float64 corners) -> float (NaN when the union is 0)."""
    parts = _nms_parts(np.asarray(ca, np.float64), np.asarray(cb, np.float64))
    if parts is None:
        return 0.0
    inter, union = parts
    return _quotient(_f32_of(inter), union - inter)


def _ulp32(v):
    return float(np.spacing(np.float32(abs(v)) * np.float32(2)))       # generous: the next binade's ulp


def _ulp64(v):
    return float(np.spacing(abs(v) * 2.0))


def _nms_eps(box, k):
    """Largest displacement of a footprint corner when cos / sin move by k ulp (0 for yaw 0: cos 1, sin 0 exact)."""
    x, y, z, l, h, w, yaw = (float(np.float32(v)) for v in box)
    if yaw == 0.0:
        return 0.0
    c, s = nms_trig(yaw)
    return math.sqrt(2.0) * k * (abs(l) / 2 * _ulp32(c) + abs(w) / 2 * _ulp32(s)) + 8 * _U * (abs(x) + abs(z) + abs(l) + abs(w))


def _fp_slack(pts_a, pts_b):
    """Absolute bound of the fp64 rounding of a clipper's areas (products of coordinates of magnitude R)."""
    r = float(np.abs(np.concatenate([np.asarray(pts_a).reshape(-1), np.asarray(pts_b).reshape(-1)])).max())
    return 256 * _U * (r * r + 1.0)


def _fast_parts(fa, fb):
    """(shared, area a, area b) of two footprints by the float64 clipper: the slopes of the perturbation."""
    from oracle.postprocess import clip_convex, polygon_area
    aa, ab = polygon_area(fa), polygon_area(fb)
    shared = polygon_area(clip_convex(fa, fb)) if aa > 0 and ab > 0 else 0.0
    return np.array([shared, aa, ab])


def _spread(footprint_a, footprint_b, trig_a, trig_b, ulp, k):
    """Linearised spread of (shared, area a, area b) when each of the four trig values moves by +-k ulp: twice the
    sum over the values of the larger one-sided change (the slopes are measured with the float64 clipper, whose
    rounding is far below the change of a few ulp of the trig)."""
    base = _fast_parts(footprint_a(trig_a), footprint_b(trig_b))
    total = np.zeros(3)
    for which, trig in ((0, trig_a), (1, trig_b)):
        if trig is None:
            continue
        for j in range(2):
            worst = np.zeros(3)
            for sign in (1, -1):
                t = list(trig)
                t[j] += sign * k * ulp(t[j])
                ta, tb = (t, trig_b) if which == 0 else (trig_a, t)
                worst = np.maximum(worst, np.abs(_fast_parts(footprint_a(ta), footprint_b(tb)) - base))
            total += worst
    return 2.0 * total


def _widen(lo, hi):
    """A few ulp more on each side: the final subtraction and division of the fp64 code."""
    return lo - 8 * _U * abs(lo), hi + 8 * _U * abs(hi)


def nms_iou_interval(box_a, box_b, k=TRIG_ULPS, appr=None, exact_fp=False):
    """(lo, hi) enclosing nms.py:64-88's IoU of float32 boxes a (single box) and b over cos / sin moved by up to k ulp
    and the kernel's fp64 rounding (exact_fp: the configuration is computed exactly, e.g. yaw 0 with one box inside
    the other and dyadic coordinates).  appr: the int_corners path; the truncated corners are enumerated.  Returns
    (nan, nan) when the overlap may be NaN, and (-inf, inf) when too many truncations are undecided."""
    if appr is not None:
        return _int_interval(box_a, box_b, k, appr)
    ca, cb = nms_corners(box_a), nms_corners(box_b)
    fa, fb = ca[:4, [0, 2]], cb[:4, [0, 2]]
    slack = 0.0 if exact_fp else _fp_slack(fa, fb)
    ta = None if float(np.float32(box_a[6])) == 0.0 else nms_trig(box_a[6])
    tb = None if float(np.float32(box_b[6])) == 0.0 else nms_trig(box_b[6])
    if ta is None and tb is None and slack == 0:
        v = nms_iou(ca, cb)
        return v, v
    e = _nms_eps(box_a, k) + _nms_eps(box_b, k)
    mx0, mn0, mx, mn = ca.max(0), ca.min(0), cb.max(0), cb.min(0)
    if np.any((mx0 + e < mn) | (mn0 - e > mx)):          # apart under every perturbation: the early-out
        return 0.0, 0.0
    maybe_apart = bool(np.any((mx0 - e < mn) | (mn0 + e > mx)))
    spread = _spread(lambda t: nms_corners(box_a, t)[:4, [0, 2]], lambda t: nms_corners(box_b, t)[:4, [0, 2]],
                     ta, tb, lambda v: _ulp32(v), k) + slack
    f = Fraction
    s_sh, s_a, s_b = (f(float(v)) for v in spread)
    ha, hb = f(mx0[1]) - f(mn0[1]), f(mx[1]) - f(mn[1])
    shared_y = max(f(0), min(f(mx[1]), f(mx0[1])) - max(f(mn[1]), f(mn0[1])))
    inter = shared_y * intersection_area(fa, fb)
    union = hb * area(fb) + ha * area(fa)
    lo_i, hi_i = max(f(0), inter - shared_y * s_sh), inter + shared_y * s_sh
    lo_u, hi_u = union - hb * s_b - ha * s_a, union + hb * s_b + ha * s_a
    if lo_u - hi_i <= 0:
        return math.nan, math.nan
    lo, hi = _widen(_quotient(_f32_of(lo_i), hi_u - lo_i), _quotient(_f32_of(hi_i), lo_u - hi_i))
    return (min(lo, 0.0) if maybe_apart else lo), hi


def _int_interval(box_a, box_b, k, appr, limit=8):
    """nms_iou_interval on np.int32(corners * appr): every truncation that can flip is enumerated."""
    options = []
    for box in (box_a, box_b):
        base = nms_corners(box)
        eps = _nms_eps(box, k)
        lo = np.int32((base - eps) * appr).astype(np.float64)
        hi = np.int32((base + eps) * appr).astype(np.float64)
        lo[:, 1] = hi[:, 1] = np.int32(base[:, 1] * appr)
        options.append((lo, hi))
    flips = [(b, i, j) for b in range(2) for i in range(4) for j in (0, 2) if options[b][0][i, j] != options[b][1][i, j]]
    if len(flips) > limit:
        return -math.inf, math.inf
    values = []
    for mask in range(1 << len(flips)):
        corners = [options[0][0].copy(), options[1][0].copy()]
        for bit, (b, i, j) in enumerate(flips):
            if mask >> bit & 1:
                corners[b][i, j] = options[b][1][i, j]
        for b in range(2):
            corners[b][4:, [0, 2]] = corners[b][:4, [0, 2]]
        values.append(nms_iou(corners[0], corners[1]))
    if any(math.isnan(v) for v in values):
        return math.nan, math.nan
    # integer corners: only the intersection points of rotated edges carry fp64 rounding
    rot = any(float(np.float32(b[6])) != 0.0 for b in (box_a, box_b))
    pad = 1e-12 if rot else 0.0
    return min(values) * (1 - pad), max(values) * (1 + pad)


# ---------------------------------------------------------------------------------------------
# KITTI evaluator: toPolygon (:265-288), groundBoxOverlap / box3DOverlap / imageBoxOverlap
# ---------------------------------------------------------------------------------------------
def eval_footprint(l, w, t1, t3, ry, trig=None):
    """toPolygon in double: [4, 2] (x, z) corners (trig overrides (cos ry, sin ry))."""
    c, s = (math.cos(ry), math.sin(ry)) if trig is None else trig
    lx, lz = [l / 2, l / 2, -l / 2, -l / 2], [w / 2, -w / 2, -w / 2, w / 2]
    return np.array([[(c * lx[i] + s * lz[i]) + t1, (-s * lx[i] + c * lz[i]) + t3] for i in range(4)])


def _row_fp(g):
    """(l, w, t1, t3, ry) of a ground-truth [14] or detection [15] row (both put h, w, l, t1, t2, t3, ry last)."""
    return g[9], g[8], g[10], g[12], g[13]


def _eval_parts(g, d):
    gp, dp = eval_footprint(*_row_fp(g)), eval_footprint(*_row_fp(d))
    return gp, dp, intersection_area(gp, dp), area(gp), area(dp)


def ground_overlap(g, d, criterion=-1):
    """groundBoxOverlap(d, g, criterion) of a ground-truth row g [14] and a detection row d [15]."""
    _, _, inter, ga, da = _eval_parts(g, d)
    return _quotient(inter, ga + da - inter if criterion == -1 else da)


def _vols(g, d):
    """box3DOverlap's height overlap and volumes: t2 - h and the volume products are double, as there."""
    ymax = min(g[11], d[11])
    ymin = max(d[11] - d[7], g[11] - g[7])
    det_vol = d[7] * d[9] * d[8]
    gt_vol = g[7] * g[9] * g[8]
    return max(Fraction(0), Fraction(ymax) - Fraction(ymin)), Fraction(det_vol), Fraction(gt_vol)


def box3d_overlap(g, d, criterion=-1):
    """box3DOverlap(d, g, criterion)."""
    _, _, inter, _, _ = _eval_parts(g, d)
    dy, det_vol, gt_vol = _vols(g, d)
    inter_vol = inter * dy
    return _quotient(inter_vol, det_vol + gt_vol - inter_vol if criterion == -1 else det_vol)


def image_overlap(d, g, criterion=-1):
    """imageBoxOverlap(d, g, criterion) on the [x1, y1, x2, y2] boxes of the rows (columns 3-6 of both)."""
    f = Fraction
    a, b = [f(v) for v in d[3:7]], [f(v) for v in g[3:7]]
    w = min(a[2], b[2]) - max(a[0], b[0])
    h = min(a[3], b[3]) - max(a[1], b[1])
    if w <= 0 or h <= 0:
        return 0.0
    inter = w * h
    a_area = (a[2] - a[0]) * (a[3] - a[1])
    b_area = (b[2] - b[0]) * (b[3] - b[1])
    return _quotient(inter, a_area + b_area - inter if criterion == -1 else a_area)


def eval_overlap_interval(g, d, metric, criterion=-1, k=TRIG_ULPS, exact_fp=False):
    """(lo, hi) enclosing the ground (metric 1) or 3D (metric 2) overlap over cos / sin moved by up to k ulp and the
    fp64 rounding of the clippers (exact_fp: computed exactly)."""
    gp, dp, inter, ga, da = _eval_parts(g, d)
    lg, wg, xg, zg, rg = _row_fp(g)
    ld, wd, xd, zd, rd = _row_fp(d)
    slack = 0.0 if exact_fp else _fp_slack(gp, dp)
    tg = None if rg == 0.0 else (math.cos(rg), math.sin(rg))
    td = None if rd == 0.0 else (math.cos(rd), math.sin(rd))
    if tg is None and td is None and slack == 0:
        v = ground_overlap(g, d, criterion) if metric == 1 else box3d_overlap(g, d, criterion)
        return v, v
    spread = _spread(lambda t: eval_footprint(lg, wg, xg, zg, rg, t), lambda t: eval_footprint(ld, wd, xd, zd, rd, t),
                     tg, td, _ulp64, k) + slack
    s_i, sg, sd = (Fraction(float(v)) for v in spread)
    lo_i, hi_i = max(Fraction(0), inter - s_i), inter + s_i
    if metric == 1:
        if criterion == -1:
            bounds = _quotient(lo_i, ga + da + sg + sd - lo_i), _quotient(hi_i, ga + da - sg - sd - hi_i)
        else:
            bounds = _quotient(lo_i, da + sd), _quotient(hi_i, da - sd)
    else:
        dy, det_vol, gt_vol = _vols(g, d)
        if criterion == -1:
            bounds = _quotient(lo_i * dy, det_vol + gt_vol - lo_i * dy), _quotient(hi_i * dy, det_vol + gt_vol - hi_i * dy)
        else:
            bounds = _quotient(lo_i * dy, det_vol), _quotient(hi_i * dy, det_vol)
    return _widen(*bounds)


def decide(interval, thres):
    """True: the value is certainly > thres; False: certainly <= thres; None: the interval straddles thres (or NaN)."""
    lo, hi = interval
    if math.isnan(lo) or math.isnan(hi):
        return None
    if lo > thres:
        return True
    if hi <= thres:
        return False
    return None

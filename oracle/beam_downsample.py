"""CPU oracle of the LiDAR beam downsampling tool (reference scripts/point_cloud_downsample.py:19-53).

TEST INFRASTRUCTURE (see oracle/__init__.py).

* ``cosines`` / ``band_mask`` / ``downsample`` - a NumPy restatement of the script's arithmetic: the float32 norm,
  the float64 cosine, the float64 band limits between the sorted centres and the kept rows in original order.
  tests/test_beam_downsample_cpu.py checks it against the bytes the reference's own script wrote
  (tests/golden/beam_downsample.npz, made by ``tools/make_golden.py beam_downsample``).
* ``exact_kmeans_1d`` - the exact 1-D k-means: k divide-and-conquer DP layers over the sorted values, vectorised
  per recursion level, with the cost of a group from double-double prefix sums of the values minus the first one.
  The double-double operations are the same sequence of rounded operations ``csrc/pg_beam.cu`` performs (Dekker's
  product here where the kernel uses an FMA: both give the exact rounding error); the prefix sums are accumulated
  in order here and per chunk there, so the two can differ in the last bits of a cost.  Ties go to the smallest
  split index.  It counts near-ties: decisions where another split's total lies within ``tol`` (relative) of the
  best one, where a last-bit difference could change the choice.  Fast enough for frames of about 20 000 points.
* ``velodyne_frame`` - a seeded synthetic velodyne-coordinate frame (oracle/synth.py's scene mapped through the
  calibration of oracle/kitti.py), [M, 4] float32 rows as in a .bin file.
"""
import math
import os
import tempfile

import numpy as np


# ---- the reference script's arithmetic ----

def cosines(xyz):
    """:22-25 and :29, the float64 zenith cosine of every point (NaN / inf where the norm is zero)."""
    xyz = np.asarray(xyz, dtype=np.float32)
    with np.errstate(divide='ignore', invalid='ignore'):
        xyz_norm = np.sqrt(np.sum(xyz * xyz, axis=1, keepdims=True))
        z_axis = np.array([[0], [0], [1]])
        cos = xyz.dot(z_axis) / xyz_norm
    return cos.reshape(-1)


def band_mask(cos, centers, downsample_rate):
    """:27-35, with the centres sorted as :27 does."""
    centers = [-1, ] + np.sort(np.asarray(centers, dtype=np.float64).reshape(-1)).tolist() + [1, ]
    mask = np.zeros(len(cos), dtype=bool)
    with np.errstate(invalid='ignore'):
        for i in range(0, len(centers) - 2, downsample_rate):
            lower = (centers[i] + centers[i + 1]) / 2
            higher = (centers[i + 1] + centers[i + 2]) / 2
            mask += (cos > lower) * (cos < higher)
    return mask


def downsample(velo, centers, downsample_rate):
    """:20-53 for one frame's [M, 4] float32 rows and its centres -> the [R, 4] float32 rows the script writes."""
    velo = np.asarray(velo, dtype=np.float32).reshape(-1, 4)
    mask = band_mask(cosines(velo[:, :3]), centers, downsample_rate)
    return np.hstack([velo[:, :3][mask, :], velo[:, [3]][mask, :]])


# ---- double-double arithmetic (vectorised; same operation sequence as pg_beam.cu) ----

def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _fast_two_sum(a, b):
    s = a + b
    return s, b - (s - a)


def _split(a):
    c = 134217729.0 * a
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _dd_add(xh, xl, yh, yl):
    sh, sl = _two_sum(xh, yh)
    th, tl = _two_sum(xl, yl)
    sh, sl = _fast_two_sum(sh, sl + th)
    return _fast_two_sum(sh, sl + tl)


def _dd_sub(xh, xl, yh, yl):
    return _dd_add(xh, xl, -yh, -yl)


def _dd_mul(xh, xl, yh, yl):
    p, e = _two_prod(xh, yh)
    return _fast_two_sum(p, e + (xh * yl + xl * yh))


def _dd_div(xh, xl, n):
    q1 = xh / n
    p, pe = _two_prod(q1, n)
    rh, _ = _dd_sub(xh, xl, p, pe)
    return _fast_two_sum(q1, rh / n)


def prefix_sums(x):
    """Double-double prefix sums [n + 1] of e_i = x_i - x_0 (exact) and e_i^2, accumulated in order."""
    n = len(x)
    s = np.zeros((4, n + 1), dtype=np.float64)
    if n == 0:
        return s
    eh, el = _two_sum(x, -x[0])
    qh, ql = _dd_mul(eh, el, eh, el)
    a1h = a1l = a2h = a2l = 0.0
    for i in range(n):
        a1h, a1l = _dd_add(a1h, a1l, float(eh[i]), float(el[i]))
        a2h, a2l = _dd_add(a2h, a2l, float(qh[i]), float(ql[i]))
        s[0, i + 1], s[1, i + 1], s[2, i + 1], s[3, i + 1] = a1h, a1l, a2h, a2l
    return s


def group_cost(x, s, a, b):
    """cost of the groups [a, b) of the sorted values x (arrays of split pairs, a < b)."""
    a = np.asarray(a, dtype=np.int64)
    b = np.asarray(b, dtype=np.int64)
    d1h, d1l = _dd_sub(s[0, b], s[1, b], s[0, a], s[1, a])
    d2h, d2l = _dd_sub(s[2, b], s[3, b], s[2, a], s[3, a])
    qh, ql = _dd_mul(d1h, d1l, d1h, d1l)
    qh, ql = _dd_div(qh, ql, (b - a).astype(np.float64))
    c, _ = _dd_sub(d2h, d2l, qh, ql)
    c = np.where(c > 0.0, c, 0.0)
    return np.where(x[a] == x[b - 1], 0.0, c)


def exact_kmeans_1d(values, k, tol=1e-12):
    """The exact 1-D k-means of the finite entries of ``values`` -> dict(centers [k] ascending group means,
    inertia, sizes [k] group sizes in sorted order, near_ties: number of DP decisions with a near-tie).
    No finite value: NaN centres, zero inertia.  1 <= finite values < k: ValueError."""
    v = np.asarray(values, dtype=np.float64).reshape(-1)
    x = np.sort(v[np.isfinite(v)])
    n = len(x)
    if n == 0:
        return dict(centers=np.full(k, np.nan), inertia=0.0, sizes=np.zeros(k, np.int64), near_ties=0)
    if n < k:
        raise ValueError('n_samples=%d should be >= n_clusters=%d' % (n, k))
    s = prefix_sums(x)
    f_prev = np.full(n + 1, np.nan)
    j = np.arange(1, n - k + 2)
    f_prev[j] = group_cost(x, s, np.zeros_like(j), j)
    opts = {}
    near_ties = 0
    for layer in range(2, k + 1):
        j1 = n - k + layer
        jlo, jhi = np.array([n if layer == k else layer]), np.array([j1])
        alo, ahi = np.array([layer - 1]), np.array([j1 - 1])
        opt = np.full(n + 1, -1, dtype=np.int64)
        f_cur = np.full(n + 1, np.nan)
        while True:
            live = jlo <= jhi
            jlo, jhi, alo, ahi = jlo[live], jhi[live], alo[live], ahi[live]
            if len(jlo) == 0:
                break
            jm = (jlo + jhi) >> 1
            cnt = np.minimum(ahi, jm - 1) - alo + 1
            starts = np.concatenate([[0], np.cumsum(cnt)[:-1]])
            seg = np.repeat(np.arange(len(jm)), cnt)
            a = alo[seg] + (np.arange(int(cnt.sum())) - starts[seg])
            tot = f_prev[a] + group_cost(x, s, a, jm[seg])
            mins = np.minimum.reduceat(tot, starts)
            hit = np.flatnonzero(tot == mins[seg])
            best = a[hit[np.unique(seg[hit], return_index=True)[1]]]
            m = mins[seg]
            near = (np.abs(tot - m) <= tol * np.abs(m)) & ~((tot == 0.0) & (m == 0.0))
            near_ties += int((np.add.reduceat(near.astype(np.int64), starts) > 1).sum())
            opt[jm] = best
            f_cur[jm] = mins
            jlo, jhi, alo, ahi = (np.concatenate([jlo, jm + 1]), np.concatenate([jm - 1, jhi]),
                                  np.concatenate([alo, best]), np.concatenate([best, ahi]))
        opts[layer] = opt
        f_prev = f_cur
    bounds = [n]
    for layer in range(k, 1, -1):
        bounds.append(int(opts[layer][bounds[-1]]))
    bounds.append(0)
    bounds = bounds[::-1]
    centers = np.empty(k)
    inertia = []
    for g in range(k):
        grp = x[bounds[g]:bounds[g + 1]]
        centers[g] = math.fsum(grp) / len(grp)
        inertia.append(math.fsum((grp - centers[g]) ** 2))
    return dict(centers=centers, inertia=math.fsum(inertia), sizes=np.diff(bounds).astype(np.int64),
                near_ties=near_ties)


# ---- synthetic velodyne frames ----

def velodyne_frame(seed, num_points, full_360=True):
    """oracle/synth.py's scene (64 beams) in velodyne coordinates, [num_points, 4] float32 (x, y, z, reflectance),
    mapped as oracle/kitti.write_synthetic_kitti maps its frames."""
    from . import kitti, synth
    fd, path = tempfile.mkstemp(suffix='.txt')
    try:
        with os.fdopen(fd, 'w') as f:
            f.write(kitti.CALIB_TEXT)
        calib = kitti.parse_calib(path)
    finally:
        os.remove(path)
    xyz, intensity = synth.lidar_frame(seed, num_points, full_360=full_360)
    velo = np.matmul(np.hstack([xyz.astype(np.float64), np.ones([len(xyz), 1])]),
                     np.transpose(calib['cam_to_velo']))[:, :3]
    return np.hstack([velo, intensity]).astype(np.float32)

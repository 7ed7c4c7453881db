"""Seeded synthetic inputs: KITTI-shape LiDAR frames (SURVEY.md section 8d) and integer-valued layer cases.

TEST INFRASTRUCTURE (see oracle/__init__.py).  A 64-beam spinning LiDAR is
ray-cast against a ground plane, two side walls and 12 car-sized boxes, in the
camera frame the reference feeds its graph generator with
(x right, y down, z forward; reference dataset/kitti_dataset.py:998-1006).
Frame ``i`` uses ``numpy.random.default_rng(1000 + i)``.

The integer cases (``exact_*`` below) have weights, biases, features and coordinates so small that every route of the
library computes them exactly, whatever its summation order or arithmetic (fp32 FFMA, BF16x3, FP16): every layer
input and pre-activation is an integer of magnitude <= EXACT_VALUE (exact in FP16, and the BF16x3 split of it and its
product with a weight are exact), every dot product has sum_k |x_k w_k| + |b| < EXACT_DOT (headroom under fp32's 2^24
for the accumulator's alignment of addends), and every destination and column has sum_e |h_e| < EXACT_SUM.  The
float64 oracle (oracle/gnn.py) cast to float32 is then an exact reference, and a lost or repeated edge changes the
sum: the last layer's weights are >= 0 and its biases >= 1, so every edge adds at least 1 to every column of its
destination's sum under ReLU and ReLU6.  ``exact_margins`` checks those conditions on a case.
"""
import numpy as np

SENSOR_HEIGHT = 1.73
MAX_RANGE = 80.0


def _ray_box(d, lo, hi):
    """Slab test for rays from the origin with directions d [R,3] -> t [R] (inf = miss)."""
    with np.errstate(divide='ignore', invalid='ignore'):
        t0 = lo[None, :] / d
        t1 = hi[None, :] / d
    tmin = np.minimum(t0, t1)
    tmax = np.maximum(t0, t1)
    tn = np.nanmax(tmin, axis=1)
    tf = np.nanmin(tmax, axis=1)
    hit = (tn <= tf) & (tf > 0) & (tn > 0)
    return np.where(hit, tn, np.inf)


def lidar_frame(frame_idx=0, num_points=20000, full_360=False):
    """-> (xyz [N,3] float32, intensity [N,1] float32).

    num_points=None keeps every return (about 28 k front crop / 127 k full 360).
    """
    rng = np.random.default_rng(1000 + int(frame_idx))
    elev = np.deg2rad(np.linspace(2.0, -24.8, 64))
    azim = np.deg2rad(np.arange(2000) * (360.0 / 2000) - 180.0)
    if not full_360:
        azim = azim[np.abs(azim) < np.deg2rad(40.5)]
    az, el = np.meshgrid(azim, elev, indexing='ij')
    az = az.ravel() + rng.normal(0.0, 1e-3, az.size)
    el = el.ravel() + rng.normal(0.0, 1e-3, el.size)
    d = np.stack([np.cos(el) * np.sin(az), -np.sin(el), np.cos(el) * np.cos(az)], axis=1)
    # ground plane y = +SENSOR_HEIGHT (y points down)
    with np.errstate(divide='ignore'):
        t = np.where(d[:, 1] > 1e-9, SENSOR_HEIGHT / d[:, 1], np.inf)
    # side walls x = +-12 m, 4 m tall
    for xw in (-12.0, 12.0):
        with np.errstate(divide='ignore'):
            tw = np.where(d[:, 0] * xw > 1e-9, xw / d[:, 0], np.inf)
        yw = tw * d[:, 1]
        ok = np.isfinite(tw) & (yw <= SENSOR_HEIGHT) & (yw >= SENSOR_HEIGHT - 4.0)
        t = np.minimum(t, np.where(ok, tw, np.inf))
    # 12 axis-aligned boxes, 1.6 wide (x) x 1.5 tall (y) x 4.0 long (z), on the ground
    bx = rng.uniform(-9.0, 9.0, 12)
    bz = rng.uniform(6.0, 60.0, 12)
    if full_360:
        bz = bz * rng.choice([-1.0, 1.0], 12)
    for cx, cz in zip(bx, bz):
        lo = np.array([cx - 0.8, SENSOR_HEIGHT - 1.5, cz - 2.0])
        hi = np.array([cx + 0.8, SENSOR_HEIGHT, cz + 2.0])
        t = np.minimum(t, _ray_box(d, lo, hi))
    keep = np.isfinite(t) & (t < MAX_RANGE)
    xyz = d[keep] * t[keep, None] + rng.normal(0.0, 0.02, (int(keep.sum()), 3))
    if num_points is not None:
        if xyz.shape[0] < num_points:
            raise ValueError('scene produced only %d returns' % xyz.shape[0])
        sel = rng.choice(xyz.shape[0], size=num_points, replace=False)
        xyz = xyz[np.sort(sel)]
    xyz = xyz.astype(np.float32)
    intensity = rng.random((xyz.shape[0], 1), dtype=np.float32)
    return xyz, intensity


# ---- integer-valued layer cases ---------------------------------------------------------------------------------------
EXACT_VALUE = 1024           # |layer input|, |pre-activation|
EXACT_DOT = 1 << 20          # sum_k |x_k w_k| + |b| of one dot product
EXACT_SUM = 1 << 23          # sum_e |h_e| of one destination and column
EXACT_ACTIVATIONS = ('NONE', 'ReLU', 'ReLU6')     # the activations that keep integers integers


def exact_weights(rng, dims):
    """-> (ws, bs) float32: weights in {-2, ..., 2}, mostly 0, every row and every column of every W with a nonzero
    (so every 16-row k chunk and every column block counts); biases in {-2, ..., 2}; the last layer's weights >= 0 and
    its biases >= 1."""
    ws, bs = [], []
    for l, (k, n) in enumerate(zip(dims[:-1], dims[1:])):
        last = l == len(dims) - 2
        mask = rng.random((k, n)) < 0.01
        mask[np.arange(k), rng.integers(0, n, k)] = True
        mask[rng.integers(0, k, n), np.arange(n)] = True
        mag = np.where(rng.random((k, n)) < 0.25, 2, 1)
        sign = 1 if last else rng.choice([-1, 1], (k, n))
        ws.append(np.where(mask, sign * mag, 0).astype(np.float32))
        bs.append((rng.integers(1, 3, n) if last else rng.integers(-2, 3, n)).astype(np.float32))
    return ws, bs


def exact_edge_case(layer, dims, num_vertices, seed, coord_range=None):
    """An integer edge layer: layer 'gnn' (GraphNetAutoCenter, dims[0] = C_in + 3, destinations are the vertices,
    xyz_dst = xyz + an integer offset) or 'pool' (PointSetPooling, dims[0] = 4: one intensity channel, destinations
    are keypoints dst_index, a permutation of the points).  -> dict(layer, dims, feat, xyz, xyz_dst, dst_index, ws,
    bs), float32 arrays holding small integers.  Coordinates are in [-coord_range, coord_range] (default 4 for 'gnn' and 2
    for 'pool', which has more layers to grow through)."""
    rng = np.random.default_rng(seed)
    c_in = dims[0] - 3
    ws, bs = exact_weights(rng, dims)
    feat = np.where(rng.random((num_vertices, c_in)) < 0.3, rng.integers(1, 4, (num_vertices, c_in)), 0)
    r = coord_range if coord_range is not None else 4 if layer == 'gnn' else 2
    xyz = rng.integers(-r, r + 1, (num_vertices, 3))
    case = dict(layer=layer, dims=list(dims), ws=ws, bs=bs, feat=feat.astype(np.float32), xyz=xyz.astype(np.float32))
    if layer == 'gnn':
        case['xyz_dst'] = (xyz + rng.integers(-1, 2, xyz.shape)).astype(np.float32)
        case['dst_index'] = None
    else:
        assert layer == 'pool' and c_in == 1, (layer, dims)
        case['xyz_dst'] = case['xyz']
        case['dst_index'] = rng.permutation(num_vertices).astype(np.int32)
    return case


def edges_from_degrees(rng, degrees, num_src):
    """The edge list whose destination runs are given: destination d owns `degrees[d]` consecutive rows, in
    destination order; sources uniform in [0, num_src).  -> (src, dst) int32."""
    dst = np.repeat(np.arange(len(degrees)), degrees).astype(np.int32)
    return rng.integers(0, num_src, dst.size).astype(np.int32), dst


def _fill(rng, total, high=40):
    """Random degrees in [1, high] summing to exactly total (>= 0)."""
    out = []
    while total > 0:
        d = int(min(total, rng.integers(1, high + 1)))
        out.append(d)
        total -= d
    return out


ORDERED_SLICE = 1 << 18       # edges per launch and fix-up of the ordered segment sum (pg_common.cuh kOrderedSlice)
STORE_SLICE = 1 << 20         # stored rows per slice of the pooling split's last layer (pg_tc.cu launch_edge)
TAIL_SIZES = (1, 15, 16, 17, 63, 64, 65, 191, 192, 193)


def exact_edge_list(name, seed=0):
    """-> dict(name, src, dst, num_dst, marks): an edge list grouped by destination (num_src = num_dst vertices);
    marks: the rows it is built around.

    mixed       ~55 k edges: in-degrees 0 .. 40, a hub of degree 3000, empty destinations in the middle and past the
                last edge, E not a multiple of 16 (a partial last unit)
    slices      3 * 2^18 + 1000 edges: one destination starts mid-unit before row 2^18 and ends mid-unit after row
                2 * 2^18 (degree > 2^18: it straddles the first slice boundary and covers the whole second slice and
                both its boundaries); a run ends exactly at row 3 * 2^18 - 1 and a degree-1 destination follows
    pool_slices 2^20 + 2^18 + 5 edges: one destination straddles stored row 2^20, mid-unit at both ends
    tail_<E>    E edges over about E / 3 destinations, some empty
    """
    rng = np.random.default_rng(seed + 7 * len(name))
    S = ORDERED_SLICE
    marks = {}
    if name == 'mixed':
        deg = rng.integers(0, 41, 2600)
        deg[1234] = 3000
        deg[[17, 900, 1800]] = 0
        deg[-5:] = 0
        while deg.sum() % 16 == 0:
            deg[2000] = deg[2000] % 40 + 1
        marks = dict(hub=1234, empty=[17, 900, 1800, 2599])
    elif name == 'slices':
        deg = _fill(rng, S - 37)
        big = len(deg)
        deg.append((2 * S + 21) - (S - 37))
        deg += _fill(rng, 3 * S - (2 * S + 21))
        ends = len(deg) - 1
        deg.append(1)
        deg += _fill(rng, 999) + [0, 0, 0]
        deg = np.array(deg)
        marks = dict(big=big, ends_at_slice=ends, single=ends + 1)
    elif name == 'pool_slices':
        P = STORE_SLICE
        deg = _fill(rng, P - 29)
        straddle = len(deg)
        deg.append(29 + 43)
        deg += _fill(rng, S + 5 - 43) + [0]
        deg = np.array(deg)
        marks = dict(straddle=straddle)
    elif name.startswith('tail_'):
        e = int(name[5:])
        num_dst = e // 3 + 3
        deg = np.bincount(rng.integers(0, num_dst - 1, e), minlength=num_dst)
    else:
        raise KeyError(name)
    src, dst = edges_from_degrees(rng, deg, len(deg))
    return dict(name=name, src=src, dst=dst, num_dst=len(deg), marks=marks)


def exact_edge_inputs(case, src, dst):
    """The first layer's input rows of edges (src, dst) in float64: [features[src], xyz[src] - xyz_dst[row(dst)]]."""
    drow = dst if case['dst_index'] is None else case['dst_index'][dst]
    return np.concatenate([case['feat'][src], case['xyz'][src] - case['xyz_dst'][drow]], axis=1).astype(np.float64)


def exact_edge_reference(case, edges, act, aggregation, dtype=np.float64, fp16=False):
    """oracle.gnn's edge layer on the case's inputs in `dtype` (fp16: the FP16 oracle), cast to float32."""
    from oracle import gnn as ognn
    c = {k: (case[k].astype(dtype) if k in ('feat', 'xyz', 'xyz_dst') else case[k]) for k in case}
    ws, bs = [w.astype(dtype) for w in case['ws']], [b.astype(dtype) for b in case['bs']]
    src, dst, num_dst = edges['src'], edges['dst'], edges['num_dst']
    if case['layer'] == 'gnn':
        out = ognn.gnn_edge_layer(c['feat'], c['xyz'], c['xyz_dst'], src, dst, num_dst, ws, bs, act=act,
                                  aggregation=aggregation, fp16=fp16)
    else:
        out = ognn.pool_edge_layer(c['feat'], c['xyz'], c['xyz_dst'][case['dst_index']], src, dst, num_dst, ws, bs,
                                   act=act, aggregation=aggregation, fp16=fp16)
    return out.astype(np.float32)


def _layer_margins(x, ws, bs, acts, worst):
    """Run integer rows x (float64) through the layers, updating worst's ratios; -> the last layer's output.  Integer
    inputs and weights keep every value an integer under EXACT_ACTIVATIONS (float64 is exact far beyond these bounds),
    so only the inputs are checked for it.  The dot ratio is an upper bound: sum_k max_rows|x_k| |w_k| + |b|."""
    from oracle.gnn import activate
    worst['integer'] &= bool(np.array_equal(x, np.rint(x)))
    for w, b, act in zip(ws, bs, acts):
        w, b = w.astype(np.float64), b.astype(np.float64)
        xmax = np.abs(x).max(axis=0) if len(x) else np.zeros(x.shape[1])
        worst['value'] = max(worst['value'], float(xmax.max(initial=0)) / EXACT_VALUE)
        worst['dot'] = max(worst['dot'], float((xmax @ np.abs(w) + np.abs(b)).max(initial=0)) / EXACT_DOT)
        pre = x @ w
        pre += b
        if len(pre):
            worst['value'] = max(worst['value'], max(float(pre.max()), -float(pre.min())) / EXACT_VALUE)
        x = activate(act, pre)
    return x


def _check_weights(ws, bs):
    """The weight conditions: integers in [-2, 2], a nonzero in every row and column, last layer >= 0, bias >= 1."""
    ok = True
    for w, b in zip(ws, bs):
        ok &= bool(np.all(w == np.round(w)) and np.abs(w).max() <= 2 and np.all(b == np.round(b)))
        ok &= bool(np.all((w != 0).any(axis=0)) and np.all((w != 0).any(axis=1)))
    return ok and bool(np.all(ws[-1] >= 0) and np.all(bs[-1] >= 1))


def exact_margins(case, edges, act, chunk=1 << 16):
    """The exactness conditions of an edge case on an edge list, checked in float64 layer by layer.  -> dict(
    integer: every value an integer, weights: the weight conditions hold, value / dot / sum: the worst ratio of
    max|value| to EXACT_VALUE, of sum_k |x_k w_k| + |b| to EXACT_DOT, of sum_e |h_e| to EXACT_SUM).  The case is
    exact when integer and weights are True and every ratio is < 1."""
    assert act in EXACT_ACTIVATIONS, act
    worst = dict(integer=True, weights=_check_weights(case['ws'], case['bs']), value=0.0, dot=0.0, sum=0.0)
    src, dst, num_dst = edges['src'], edges['dst'], edges['num_dst']
    acc = np.zeros((num_dst, case['dims'][-1]))
    for s in range(0, len(src), chunk):
        x = exact_edge_inputs(case, src[s:s + chunk], dst[s:s + chunk])
        h = _layer_margins(x, case['ws'], case['bs'], [act] * len(case['ws']), worst)
        _add_rows(acc, dst[s:s + chunk], np.abs(h))
    worst['sum'] = float(acc.max(initial=0)) / EXACT_SUM
    return worst


def _add_rows(acc, rows, h):
    """acc[rows] += h with repeated rows (as a sparse product: exact in float64 for these integers)."""
    from scipy import sparse
    sel = sparse.csr_matrix((np.ones(len(rows)), (rows, np.arange(len(rows)))), shape=(acc.shape[0], len(rows)))
    acc += sel @ h


def exact_dense_case(m, dims, seed, residual=False):
    """Integer dense layers: x [m, dims[0]] in {-3, ..., 3}, the weights of exact_weights, a residual [m, dims[-1]] in
    {-3, ..., 3} or None.  -> dict(x, ws, bs, residual)."""
    rng = np.random.default_rng(seed)
    ws, bs = exact_weights(rng, dims)
    x = np.where(rng.random((m, dims[0])) < 0.5, rng.integers(-3, 4, (m, dims[0])), 0).astype(np.float32)
    res = rng.integers(-3, 4, (m, dims[-1])).astype(np.float32) if residual else None
    return dict(x=x, ws=ws, bs=bs, residual=res)


def exact_dense_margins(case, acts):
    """exact_margins for dense layers with activations acts (one per layer); 'sum' is the residual's addition."""
    worst = dict(integer=True, weights=_check_weights(case['ws'], case['bs']), value=0.0, dot=0.0, sum=0.0)
    h = _layer_margins(case['x'].astype(np.float64), case['ws'], case['bs'], acts, worst)
    if case['residual'] is not None:
        worst['sum'] = float(np.abs(h + case['residual']).max()) / EXACT_SUM
    return worst


def exact_dense_reference(case, acts, dtype=np.float64, fp16=False):
    """oracle.gnn.dense layer by layer in `dtype` (fp16: the FP16 routing), plus the residual, cast to float32."""
    from oracle import gnn as ognn
    x = case['x'].astype(dtype)
    for w, b, act in zip(case['ws'], case['bs'], acts):
        x = ognn.dense(x, w.astype(dtype), b.astype(dtype), act, fp16=fp16)
        x = x.astype(dtype)
    if case['residual'] is not None:
        x = x + case['residual'].astype(dtype)
    return x.astype(np.float32)

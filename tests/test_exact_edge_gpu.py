"""Every route of the fused edge layers, the scatter ops and the dense layers compared with `==` against the float64
oracle, on the integer cases of oracle/synth.py (proved exact in test_exact_cases_cpu.py): there every route computes
exactly, whatever its summation order or arithmetic, so a lost, repeated or misplaced edge, row or column shows.

Edge layers: the GNN edge layer at n = 300, 256, 192 and 64 (152x2, 128x2, 96x2 and 64x1 column groups) and with a
512-wide hidden layer (64-wide column blocks), the car and ped pooling chains (ped: the last layer split off and
stored per edge), at fp32, BF16x3 and FP16, ReLU, ReLU6 and (pooling) linear; max, sum and mean, the sum and the
mean with torch.use_deterministic_algorithms off (atomics) and on (the ordered sum: a launch and a fix-up per 2^18
edges, and the split's stored rows in slices of 2^20).  Besides the values each call checks the route it took: the
tensor-core edge launches move exactly when oracle.gnn says the layer runs on the tensor cores, and the fix-ups count
the ordered slices.  An empty destination is exactly -FLT_MAX (max) or 0 (sum, mean); `==` ignores only the sign of
zero, which exact arithmetic does not fix."""
import contextlib

import numpy as np
import pytest
import torch

from oracle import gnn as ognn
from oracle import synth
from test_exact_cases_cpu import (DENSE_SHAPES, EDGE_CASES, case_id, dense_case, edge_case, edge_list, lists_of)

pytestmark = pytest.mark.gpu
PRECISIONS = ['fp32', 'bf16x3', 'fp16']
CODES = {'fp32': 0, 'bf16x3': 1, 'fp16': 2}
FLT_LOWEST = np.finfo(np.float32).min
# (aggregation, torch.use_deterministic_algorithms)
AGG_MODES = [('max', False), ('max', True), ('sum', False), ('sum', True), ('mean', False), ('mean', True)]


def _lib():
    from pointgnn_b200 import _lib
    return _lib


def _prec(precision):
    if precision != 'fp32' and not _lib().tc_available():
        pytest.skip('tensor-core path needs an sm_90 device')
    return CODES[precision]


def _act_code(act):
    return getattr(_lib(), {'NONE': 'PG_ACT_NONE', 'ReLU': 'PG_ACT_RELU', 'ReLU6': 'PG_ACT_RELU6'}[act])


@contextlib.contextmanager
def deterministic(on):
    was, was_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=was_warn)


def _cuda(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def _assert_equal(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = got != want
    if bad.any():
        r, c = np.argwhere(bad)[0]
        raise AssertionError('%s: %d of %d values differ; first at (%d, %d): got %r, want %r'
                             % (what, int(bad.sum()), bad.size, r, c, float(got[r, c]), float(want[r, c])))


# ---- the edge layers ------------------------------------------------------------------------------------------------
_refs = {}


def reference(layer, dims, name, act, aggregation):
    """The float64 oracle cast to float32, once per module (by exactness it is every precision's); an empty
    destination of the max is the lowest float, as unsorted_segment_max gives it in float32."""
    key = (layer, tuple(dims), name, act, aggregation)
    if key not in _refs:
        edges = edge_list(name)
        want = synth.exact_edge_reference(edge_case(layer, dims, name), edges, act, aggregation)
        if aggregation == 'max':
            want[np.bincount(edges['dst'], minlength=edges['num_dst']) == 0] = FLT_LOWEST
        _refs[key] = want
    return _refs[key]


def uses_tc(layer, dims, act, code):
    return code != 0 and (ognn.gnn_uses_tc(dims) if layer == 'gnn' else ognn.pool_uses_tc(dims, act))


def expected_fixups(layer, dims, act, code, num_edges):
    """Fix-ups of one ordered sum: one per slice of 2^18 edges; the pooling split slices its stored rows by 2^20
    first and each of those by 2^18."""
    S, P = synth.ORDERED_SLICE, synth.STORE_SLICE
    if num_edges == 0:
        return 0
    if layer == 'pool' and uses_tc(layer, dims, act, code) and dims[-1] > ognn.MAX_NT and len(dims) > 3:
        return sum(-(-min(P, num_edges - s) // S) for s in range(0, num_edges, P))
    return -(-num_edges // S)


def _inputs(case, edges, src=None, dst=None):
    lib = _lib()
    src = edges['src'] if src is None else src
    dst = edges['dst'] if dst is None else dst
    di = case['dst_index']
    return (_cuda(case['feat']), _cuda(case['xyz']), _cuda(case['xyz_dst']), None if di is None else _cuda(di),
            _cuda(src), _cuda(dst), edges['num_dst']), (lib.PG_LAYER_EDGE_GNN if case['layer'] == 'gnn'
                                                         else lib.PG_LAYER_EDGE_POOL)


EDGE_RUNS = [(layer, dims, lst, act, p) for layer, dims, lst, acts in EDGE_CASES for act in acts for p in PRECISIONS]


@pytest.mark.parametrize('layer,dims,lst,act,precision', EDGE_RUNS,
                         ids=['%s-%s-%s' % (case_id(*r[:3]), r[3], r[4]) for r in EDGE_RUNS])
def test_edge_layer_exact(layer, dims, lst, act, precision):
    """A prepared layer on every list of the entry, every aggregation, the switch off and on."""
    lib = _lib()
    code = _prec(precision)
    tc = uses_tc(layer, dims, act, code)
    for name in lists_of(lst):
        edges = edge_list(name)
        case = edge_case(layer, dims, name)
        wt, bt = [_cuda(w) for w in case['ws']], [_cuda(b) for b in case['bs']]
        handle = lib.PreparedLayer(_inputs(case, edges)[1], wt, bt, dims, code, _act_code(act))
        args, _ = _inputs(case, edges)
        for agg, det in AGG_MODES:
            want = reference(layer, dims, name, act, agg)
            t0, f0 = lib.tc_launch_count(0), lib.tc_launch_count(2)
            with deterministic(det):
                got = handle.edge_mlp_max(*args, aggregation=agg).cpu().numpy()
            what = '%s %s %s %s deterministic=%s' % (case_id(layer, dims, name), act, precision, agg, det)
            assert (lib.tc_launch_count(0) > t0) == tc, what
            fix = expected_fixups(layer, dims, act, code, len(edges['src'])) if det and agg != 'max' else 0
            assert lib.tc_launch_count(2) - f0 == fix, what
            _assert_equal(got, want, what)


MIXED_RUNS = [r for r in EDGE_RUNS if r[2] == 'mixed']


@pytest.mark.parametrize('layer,dims,lst,act,precision', MIXED_RUNS,
                         ids=['%s-%s-%s' % (case_id(*r[:3]), r[3], r[4]) for r in MIXED_RUNS])
def test_edge_layer_any_order_and_entry(layer, dims, lst, act, precision):
    """The mixed list in random order (the switch off and on, with and without the trusted flag) and the per-call
    entry: the same exact sums, means and maxima."""
    lib = _lib()
    code = _prec(precision)
    edges = edge_list(lst)
    case = edge_case(layer, dims, lst)
    wt, bt = [_cuda(w) for w in case['ws']], [_cuda(b) for b in case['bs']]
    perm = np.random.default_rng(len(dims) + dims[-1]).permutation(len(edges['src']))
    args, kind = _inputs(case, edges, edges['src'][perm], edges['dst'][perm])
    handle = lib.PreparedLayer(kind, wt, bt, dims, code, _act_code(act))
    mode = 1 if layer == 'gnn' else 0
    for agg, det in AGG_MODES:
        want = reference(layer, dims, lst, act, agg)
        what = '%s %s %s %s deterministic=%s' % (case_id(layer, dims, lst), act, precision, agg, det)
        with deterministic(det):
            for trusted in (False, True):
                got = handle.edge_mlp_max(*args, trusted=trusted, aggregation=agg).cpu().numpy()
                _assert_equal(got, want, what + ' permuted, trusted=%s' % trusted)
            got = lib.edge_mlp_max(mode, *args, wt, bt, precision=code, activation=_act_code(act),
                                   aggregation=agg).cpu().numpy()
            _assert_equal(got, want, what + ' permuted, per-call entry')


# ---- the scatter ops ------------------------------------------------------------------------------------------------
SCATTER_E = 65535 * 64 + 1000     # past 65 535 chunks of 64 edges: the kernels' blockIdx.y loop goes round


@pytest.mark.parametrize('layout', ['c3', 'c4', 'c4_misaligned', 'c300'])
def test_scatter_exact(layout):
    """pg_scatter_max (3 channels: the scalar kernel; 4 aligned: vec4; 4 one float off 16 bytes: scalar) and
    pg_scatter_sum / _mean (atomic and ordered) against segment_reduce in float64, dropped ids -1 and num_centers."""
    lib = _lib()
    channels = 300 if layout == 'c300' else int(layout[1])
    e = 50000 if layout == 'c300' else SCATTER_E
    rng = np.random.default_rng(channels + e)
    num_centers = e // 40
    ids = np.sort(rng.integers(0, num_centers - 3, e)).astype(np.int32)    # the last centres stay empty
    drop = rng.choice(e, 64, replace=False)
    ids[drop[:32]] = -1
    ids[drop[32:]] = num_centers
    feat = np.where(rng.random((e, channels)) < 0.7, rng.integers(-8, 9, (e, channels)), 0).astype(np.float32)
    if layout == 'c4_misaligned':
        base = torch.zeros(e * channels + 1, device='cuda')
        ft = base[1:].view(e, channels)
        ft.copy_(_cuda(feat))
        assert ft.data_ptr() % 16 == 4
    else:
        ft = _cuda(feat)
    it = _cuda(ids)
    keep = (ids >= 0) & (ids < num_centers)
    f64, kept = feat[keep].astype(np.float64), ids[keep]
    empty = np.bincount(kept, minlength=num_centers) == 0
    assert empty.sum() >= 3
    want = ognn.segment_reduce(f64, kept, num_centers, 'max').astype(np.float32)
    want[empty] = FLT_LOWEST
    _assert_equal(lib.scatter_max(ft, it, num_centers).cpu().numpy(), want, '%s max' % layout)
    for mean in (False, True):
        want = ognn.segment_reduce(f64, kept, num_centers, 'mean' if mean else 'sum').astype(np.float32)
        for det in (False, True):
            f0 = lib.tc_launch_count(2)
            with deterministic(det):
                got = lib.scatter_sum(ft, it, num_centers, mean=mean).cpu().numpy()
            assert lib.tc_launch_count(2) - f0 == int(det)
            _assert_equal(got, want, '%s mean=%s deterministic=%s' % (layout, mean, det))


# ---- the dense layers -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('k,n', DENSE_SHAPES, ids=['%dx%d' % s for s in DENSE_SHAPES])
def test_dense_exact(k, n, precision):
    """pg_fully_connected and a PG_LAYER_MLP prepared layer, ReLU and linear, with and without the residual; the
    tensor-core dense launches move exactly when oracle.gnn.fc_uses_tc says."""
    lib = _lib()
    code = _prec(precision)
    tc = code != 0 and ognn.fc_uses_tc(k, n)
    for residual in (False, True):
        case = dense_case(k, n, residual)
        x, w, b = _cuda(case['x']), _cuda(case['ws'][0]), _cuda(case['bs'][0])
        res = None if case['residual'] is None else _cuda(case['residual'])
        handle = lib.PreparedLayer(lib.PG_LAYER_MLP, [w], [b], [k, n], code, lib.PG_ACT_RELU)
        for act in ('ReLU', 'NONE'):
            want = synth.exact_dense_reference(case, [act])
            what = 'dense %dx%d %s %s residual=%s' % (k, n, precision, act, residual)
            t1 = lib.tc_launch_count(1)
            got = lib.fully_connected(x, w, b, act == 'ReLU', residual=res, precision=code).cpu().numpy()
            assert (lib.tc_launch_count(1) > t1) == tc, what
            _assert_equal(got, want, what + ' fully_connected')
            got = handle.mlp(x, last_linear=act == 'NONE', residual=res).cpu().numpy()
            _assert_equal(got, want, what + ' prepared')

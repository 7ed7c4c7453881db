"""The ordered segment sum and mean (PG_FLAG_DETERMINISTIC) under torch.use_deterministic_algorithms(True):
pg_scatter_sum / _mean bit for bit against a NumPy float32 restatement of their documented order, the fused edge
layers and the whole model bit-identical from call to call (also while another stream keeps the GPU busy, so that
the blocks are scheduled differently), within test_aggregation_gpu's bounds of the oracles, edge lists in any order
(the call sorts them by destination first), and with the switch off no fix-up."""
import contextlib

import numpy as np
import pytest
import torch

from test_aggregation_gpu import PRECISIONS, _cuda, _err, _layer_case, _predict, _prec, _reference, _run

pytestmark = pytest.mark.gpu


def _lib():
    from pointgnn_b200 import _lib
    return _lib


@contextlib.contextmanager
def deterministic(on=True, warn_only=False):
    was, was_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=was_warn)


@contextlib.contextmanager
def busy_stream():
    """A second stream runs a long chain of element-wise kernels (tens of ms; no cuBLAS, which the deterministic
    mode refuses without a workspace setting) while the body issues its work on the current stream."""
    side = torch.cuda.Stream()
    a = torch.randn(1 << 26, device='cuda')
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        for _ in range(200):
            a = torch.sin(a)
    try:
        yield
    finally:
        torch.cuda.synchronize()


def _degrees(rng, num_dst):
    """In-degrees 1 (most), 40 (well over a 16-edge unit), 700 and 3000 (dozens of units and 64-edge tiles), 0."""
    deg = rng.integers(1, 4, num_dst)
    deg[::7] = 1
    deg[3] = 0
    deg[5] = 40
    deg[11] = 700
    deg[num_dst // 2] = 3000
    return deg


# ---- pg_scatter_sum / _mean: exact ---------------------------------------------------------------------------------
def ordered_scatter(feat, ids, num_centers, mean, tile):
    """The documented order in NumPy float32: the edges stable-sorted by id (dropped ids last), tiles of `tile` sorted
    edges, a sequential sum from 0 per destination and tile, then the tiles' partial sums one after another."""
    keep = (ids >= 0) & (ids < num_centers)
    key = np.where(keep, ids, num_centers)
    order = np.argsort(key, kind='stable')
    out = np.zeros((num_centers, feat.shape[1]), np.float32)
    count = np.zeros(num_centers, np.float32)
    for t0 in range(0, len(order), tile):
        part, cur = None, -1
        for e in list(order[t0:t0 + tile]) + [None]:
            d = -2 if e is None else int(key[e])
            if d != cur:
                if 0 <= cur < num_centers:
                    out[cur] = out[cur] + part
                cur, part = d, np.zeros(feat.shape[1], np.float32)
            if e is not None:
                part = part + feat[e]
                if d < num_centers:
                    count[d] += 1
    if mean:
        out = out / np.maximum(count, np.float32(1))[:, None]
    return out


@pytest.mark.parametrize('mean', [False, True])
@pytest.mark.parametrize('channels', [3, 37, 300])
def test_scatter_matches_the_documented_order(channels, mean):
    lib = _lib()
    rng = np.random.default_rng(channels + 10 * mean)
    num_centers = 60
    ids = np.repeat(np.arange(num_centers), _degrees(rng, num_centers)).astype(np.int32)
    ids = np.concatenate([ids, np.array([-1, num_centers, 10 ** 6], np.int32)])   # dropped, as TF does
    ids = ids[rng.permutation(ids.size)]
    feat = (rng.standard_normal((ids.size, channels)) * np.exp(rng.standard_normal((ids.size, 1)) * 3)).astype(np.float32)
    want = ordered_scatter(feat, ids, num_centers, mean, lib.PG_ORDERED_SCATTER_TILE)
    fix0 = lib.tc_launch_count(2)
    with deterministic():
        got = lib.scatter_sum(_cuda(feat), _cuda(ids), num_centers, mean=mean).cpu().numpy()
        again = lib.scatter_sum(_cuda(feat), _cuda(ids), num_centers, mean=mean).cpu().numpy()
    assert lib.tc_launch_count(2) == fix0 + 2
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.abs(got - want).max()
    assert np.array_equal(got.view(np.uint32), again.view(np.uint32))
    # the atomic route agrees to rounding
    loose = lib.scatter_sum(_cuda(feat), _cuda(ids), num_centers, mean=mean).cpu().numpy()
    assert lib.tc_launch_count(2) == fix0 + 2
    assert np.allclose(loose, want, rtol=1e-5, atol=1e-5 * np.abs(want).max())


def test_scatter_edge_cases():
    lib = _lib()
    with deterministic():
        out = lib.scatter_sum(_cuda(np.zeros((0, 4), np.float32)), _cuda(np.zeros(0, np.int32)), 5).cpu().numpy()
        assert (out == 0).all() and out.shape == (5, 4)
        feat = np.arange(12, dtype=np.float32).reshape(6, 2)
        ids = np.array([2, 2, 2, 2, 2, 2], np.int32)
        got = lib.scatter_sum(_cuda(feat), _cuda(ids), 3, mean=True).cpu().numpy()
        assert np.array_equal(got, np.array([[0, 0], [0, 0], [5, 6]], np.float32))


# ---- the fused edge layers ------------------------------------------------------------------------------------------
def _gnn_synth_case(request):
    """The car GNN layer's weights (300 outputs: two column groups) on an edge list grouped by destination with
    _degrees' in-degrees."""
    mode, kind, inputs, _, _, num_dst, ws, bs = _layer_case('gnn', request)
    rng = np.random.default_rng(9)
    dst = np.repeat(np.arange(num_dst), _degrees(rng, num_dst))
    return mode, kind, inputs, rng.integers(0, num_dst, dst.size), dst, num_dst, ws, bs


def _case(layer, request):
    return _gnn_synth_case(request) if layer == 'gnn_synth' else _layer_case(layer, request)


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('aggregation', ['sum', 'mean'])
@pytest.mark.parametrize('layer', ['gnn', 'gnn_synth', 'car_pool', 'ped_pool'])
def test_layer_bit_identical(layer, aggregation, precision, request):
    """Two prepared calls, the second while another stream is busy, and one per-call entry: the same bits, within
    test_aggregation_gpu's 1e-3 of the oracle, one fix-up per call (a slice of at most 2^18 edges)."""
    lib = _lib()
    code = _prec(precision)
    mode, kind, inputs, src, dst, num_dst, ws, bs = _case(layer, request)
    want = _reference(mode, inputs, src, dst, num_dst, ws, bs, aggregation, precision)
    slices = -(-len(src) // (1 << 18))
    fix0 = lib.tc_launch_count(2)
    with deterministic():
        first = _run(mode, kind, inputs, src, dst, num_dst, ws, bs, aggregation, code)
        with busy_stream():
            second = _run(mode, kind, inputs, src, dst, num_dst, ws, bs, aggregation, code)
        third = _run(mode, kind, inputs, src, dst, num_dst, ws, bs, aggregation, code, prepared=False)
    assert lib.tc_launch_count(2) == fix0 + 3 * slices
    assert np.array_equal(first.view(np.uint32), second.view(np.uint32))
    assert np.array_equal(first.view(np.uint32), third.view(np.uint32))
    err = _err(first, want)
    print('%s %s %s: %.3g' % (layer, aggregation, precision, err))
    assert err <= 1e-3, err
    empty = np.bincount(dst, minlength=num_dst) == 0
    assert (first[empty] == 0).all()


def test_warn_only_is_deterministic_and_silent(request, recwarn):
    code = _prec('bf16x3')
    mode, kind, inputs, src, dst, num_dst, ws, bs = _gnn_synth_case(request)
    with deterministic(warn_only=True):
        a = _run(mode, kind, inputs, src, dst, num_dst, ws, bs, 'sum', code)
        with busy_stream():
            b = _run(mode, kind, inputs, src, dst, num_dst, ws, bs, 'sum', code)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert not [w for w in recwarn if 'determin' in str(w.message).lower()]


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('aggregation', ['sum', 'mean'])
@pytest.mark.parametrize('layer', ['gnn', 'car_pool', 'ped_pool'])
def test_edge_list_in_any_order(layer, aggregation, precision, request):
    """test_aggregation_gpu's foreign edge list in random order, under the switch, on the tensor-core paths and (fp32)
    the fp32 edge kernel: within the oracle's bound, empty destinations 0, the same bits on every call, with and
    without the trusted flag, and the same bits as the list stable-sorted by dst (which the call runs).  An
    out-of-range dst still raises."""
    lib = _lib()
    code = _prec(precision)
    mode, kind, inputs, src, dst, num_dst, ws, bs = _case(layer if layer != 'gnn' else 'gnn_synth', request)
    rng = np.random.default_rng(23)
    perm = rng.permutation(len(src))
    src, dst = src[perm], dst[perm]
    want = _reference(mode, inputs, src, dst, num_dst, ws, bs, aggregation, precision)
    order = np.argsort(dst, kind='stable')
    with deterministic():
        first = _run(mode, kind, inputs, src, dst, num_dst, ws, bs, aggregation, code)
        with busy_stream():
            second = _run(mode, kind, inputs, src, dst, num_dst, ws, bs, aggregation, code, trusted=True)
        grouped = _run(mode, kind, inputs, src[order], dst[order], num_dst, ws, bs, aggregation, code)
        bad = dst.copy()
        bad[len(bad) // 3] = num_dst
        with pytest.raises(lib.PointGNNError, match='out of range'):
            _run(mode, kind, inputs, src, bad, num_dst, ws, bs, aggregation, code)
    err = _err(first, want)
    print('%s %s %s permuted: %.3g' % (layer, aggregation, precision, err))
    assert err <= 1e-3, err
    empty = np.bincount(dst, minlength=num_dst) == 0
    assert (first[empty] == 0).all()
    assert np.array_equal(first.view(np.uint32), second.view(np.uint32))
    assert np.array_equal(first.view(np.uint32), grouped.view(np.uint32))


@pytest.mark.parametrize('precision', PRECISIONS)
def test_switch_off_runs_no_fix_up(precision, request):
    """Without the switch every call makes the same launches, the same tensor-core edge launches as with it, and no
    fix-up; with it there is one fix-up (one slice here).  The two sums agree to rounding.  (That the switch-off
    launches are the parent commit's is checked outside the suite: bench.py --dump-outputs gives the same bytes.)"""
    lib = _lib()
    code = _prec(precision)
    mode, kind, inputs, src, dst, num_dst, ws, bs = _gnn_synth_case(request)
    assert not torch.are_deterministic_algorithms_enabled()
    counts = []
    for _ in range(2):
        l0, t0, f0 = lib.launch_count(), lib.tc_launch_count(0), lib.tc_launch_count(2)
        off = _run(mode, kind, inputs, src, dst, num_dst, ws, bs, 'sum', code)
        counts.append((lib.launch_count() - l0, lib.tc_launch_count(0) - t0))
        assert lib.tc_launch_count(2) == f0
    t0, f0 = lib.tc_launch_count(0), lib.tc_launch_count(2)
    with deterministic():
        on = _run(mode, kind, inputs, src, dst, num_dst, ws, bs, 'sum', code)
    assert counts[0] == counts[1]
    assert lib.tc_launch_count(0) - t0 == counts[0][1]
    assert lib.tc_launch_count(2) - f0 == 1
    assert _err(off, on) <= 1e-5


# ---- the whole model ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision', ['bf16x3', 'fp16'])
@pytest.mark.parametrize('model', ['car', 'ped'])
def test_whole_model_bit_identical(model, precision, request):
    from pointgnn_b200.models import gnn
    _prec(precision)
    g = request.getfixturevalue(model)
    with deterministic():
        l1, b1 = _predict(g, gnn.graph_scatter_sum_fn, precision)
        with busy_stream():
            l2, b2 = _predict(g, gnn.graph_scatter_sum_fn, precision)
    assert np.array_equal(l1.view(np.uint32), l2.view(np.uint32))
    assert np.array_equal(b1.view(np.uint32), b2.view(np.uint32))


def test_scatter_plug_in_follows_the_switch():
    """graph_scatter_sum_fn called on its own (the op-by-op route) is ordered under the switch too."""
    from pointgnn_b200.models import gnn
    lib = _lib()
    rng = np.random.default_rng(3)
    ids = rng.integers(0, 500, 20000).astype(np.int32)
    feat = rng.standard_normal((ids.size, 64)).astype(np.float32)
    want = ordered_scatter(feat, ids, 500, False, lib.PG_ORDERED_SCATTER_TILE)
    with deterministic():
        got = gnn.graph_scatter_sum_fn(_cuda(feat), _cuda(ids), 500).cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))

"""The segment-max epilogue of wg_gemm_kernel: a warp whose 16 rows share one destination reduce-scatters its
columns across the lanes and flushes with all 32 lanes, any other warp runs a segmented scan per 8-row half.  Max is
exact and every accumulator row depends on that row's operands only, so any edge order must give the same bits;
destination patterns that keep every warp on the segmented scan, span many tiles and CTAs, end on tile boundaries,
stay empty or are all negative are checked against NumPy fp32 at the instruction shapes 152x2 (uneven last exchange)
and 64x1."""
import numpy as np
import pytest
import torch

from oracle import gnn as ognn

pytestmark = pytest.mark.gpu
EDGES = 400000      # > 20 tiles of 128 rows per CTA on 132 SMs
FMIN = np.finfo(np.float32).min


def _lib():
    from pointgnn_b200 import _lib
    if not _lib.tc_available():
        pytest.skip('tensor-core path needs an sm_90 device')
    return _lib


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _gnn_weights(rng, c_in, d, b1_max=None, b2_max=None):
    w1 = (rng.standard_normal((c_in + 3, d)) / np.sqrt(c_in)).astype(np.float32)
    b1 = (rng.standard_normal(d) * 0.1).astype(np.float32)
    w2 = (rng.standard_normal((d, d)) / np.sqrt(d)).astype(np.float32)
    b2 = (rng.standard_normal(d) * 0.1).astype(np.float32)
    if b1_max is not None:
        b1 = np.minimum(b1, b1_max)
    if b2_max is not None:
        b2 = np.minimum(b2, b2_max)
    return w1, b1, w2, b2


def _gnn_want(f, x, xd, src, dst, nd, w1, b1, w2, b2):
    e0 = np.concatenate([f[src], x[src] - xd[dst]], axis=1)
    return ognn.graph_scatter_max_fn(np.maximum(np.maximum(e0 @ w1 + b1, 0) @ w2 + b2, 0), dst, nd)


def _gnn_layer(lib, c_in, d, w1, b1, w2, b2):
    return lib.PreparedLayer(lib.PG_LAYER_EDGE_GNN, [_cuda(w1), _cuda(w2)], [_cuda(b1), _cuda(b2)], [c_in + 3, d, d], 1)


@pytest.mark.parametrize('d', [300, 256])
def test_gnn_edge_order_does_not_change_a_bit(d):
    """Destination-sorted and randomly permuted edge lists give identical outputs (the sorted list runs almost every
    warp through the reduce-scatter, the permuted one through the segmented scan)."""
    lib = _lib()
    rng = np.random.default_rng(d)
    nv, c_in = 3000, d
    dst = np.sort(rng.integers(0, nv, EDGES))
    src = rng.integers(0, nv, EDGES)
    f = (rng.standard_normal((nv, c_in)) * 0.5).astype(np.float32)
    x = (rng.standard_normal((nv, 3)) * 20).astype(np.float32)
    layer = _gnn_layer(lib, c_in, d, *_gnn_weights(rng, c_in, d))
    perm = rng.permutation(EDGES)
    outs = [layer.edge_mlp_max(_cuda(f), _cuda(x), _cuda(x), None, _cuda(s.astype(np.int32)), _cuda(t.astype(np.int32)),
                               nv) for s, t in ((src, dst), (src[perm], dst[perm]))]
    assert (outs[0] > FMIN).any()
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize('dims', [(4, 32, 64, 128, 300), (4, 32, 64, 128, 256, 512)])
def test_pool_edge_order_does_not_change_a_bit(dims):
    """The pooling chain (ROWS producer + segment max, 512 wide as two column blocks) under a permutation."""
    lib = _lib()
    rng = np.random.default_rng(sum(dims))
    nv, nk = 5000, 1800
    ws = [_cuda((rng.standard_normal((dims[i], dims[i + 1])) / np.sqrt(dims[i])).astype(np.float32))
          for i in range(len(dims) - 1)]
    bs = [_cuda((rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32)) for i in range(len(dims) - 1)]
    dst = np.sort(rng.integers(0, nk, EDGES))
    src = rng.integers(0, nv, EDGES)
    f = _cuda(rng.random((nv, 1)).astype(np.float32))
    x = _cuda((rng.standard_normal((nv, 3)) * 20).astype(np.float32))
    kp = _cuda(rng.integers(0, nv, nk).astype(np.int32))
    layer = lib.PreparedLayer(lib.PG_LAYER_EDGE_POOL, ws, bs, list(dims), 1)
    perm = rng.permutation(EDGES)
    outs = [layer.edge_mlp_max(f, x, x, kp, _cuda(s.astype(np.int32)), _cuda(t.astype(np.int32)), nk)
            for s, t in ((src, dst), (src[perm], dst[perm]))]
    assert (outs[0] > FMIN).any()
    assert torch.equal(outs[0], outs[1])


def _runs(lengths):
    return np.repeat(np.arange(len(lengths)), lengths)


def _pattern(name, rng):
    """(dst, num_dst) of a destination-sorted edge list with >= EDGES edges."""
    if name == 'degree1':          # 16 destinations per warp: every warp takes the segmented scan
        return np.arange(EDGES), EDGES
    if name == 'long':             # one destination of 50 000 edges (391 tiles, every CTA) among short ones
        dst = np.sort(np.concatenate([rng.integers(0, 3000, EDGES - 50000), np.full(50000, 1234)]))
        return dst, 3000
    if name == 'boundaries':       # runs ending exactly on 128-row tiles and on whole rounds of 132 tiles
        block = [128, 128, 64, 64, 1, 127, 256, 127, 1, 200, 56, 128 * 132, 3, 125, 384]
        dst = _runs(block * (EDGES // sum(block) + 1))
        return dst, int(dst[-1]) + 1
    raise ValueError(name)


@pytest.mark.parametrize('d', [300, 64])
@pytest.mark.parametrize('name', ['degree1', 'long', 'boundaries'])
def test_gnn_destination_patterns(name, d):
    lib = _lib()
    rng = np.random.default_rng(len(name) * 1000 + d)
    dst, nd = _pattern(name, rng)
    nv = max(nd, 3000)
    src = rng.integers(0, nv, dst.size)
    c_in = 32
    f = (rng.standard_normal((nv, c_in)) * 0.5).astype(np.float32)
    x = (rng.standard_normal((nv, 3)) * 20).astype(np.float32)
    w = _gnn_weights(rng, c_in, d)
    want = _gnn_want(f, x, x, src, dst, nd, *w)
    got = _gnn_layer(lib, c_in, d, *w).edge_mlp_max(_cuda(f), _cuda(x), _cuda(x), None, _cuda(src.astype(np.int32)),
                                                    _cuda(dst.astype(np.int32)), nd).cpu().numpy()
    empty = want == FMIN
    assert np.array_equal(got == FMIN, empty)
    assert np.abs(got - want)[~empty].max() < 1e-3, (name, d)


@pytest.mark.parametrize('d', [300, 64])
def test_gnn_empty_and_all_negative_destinations(d):
    """Odd destinations have no edges and stay exactly -FLT_MAX; destinations 0 mod 4 see only zero edge inputs
    (self loops of zero-feature vertices), so with b1 <= 0 and b2 < 0 every pre-activation is negative and the
    output is exactly +0.0 in every column."""
    lib = _lib()
    rng = np.random.default_rng(d + 7)
    nd, c_in = 4000, 32
    dst = np.sort(rng.integers(0, nd // 2, EDGES) * 2)
    zero = dst % 4 == 0
    src = np.where(zero, dst, rng.integers(0, nd, EDGES))
    f = (rng.standard_normal((nd, c_in)) * 0.5).astype(np.float32)
    f[::4] = 0
    x = (rng.standard_normal((nd, 3)) * 20).astype(np.float32)
    w = _gnn_weights(rng, c_in, d, b1_max=0.0, b2_max=-0.01)
    want = _gnn_want(f, x, x, src, dst, nd, *w)
    got = _gnn_layer(lib, c_in, d, *w).edge_mlp_max(_cuda(f), _cuda(x), _cuda(x), None, _cuda(src.astype(np.int32)),
                                                    _cuda(dst.astype(np.int32)), nd).cpu().numpy()
    assert (got[1::2] == FMIN).all()
    neg = np.unique(dst[zero])
    assert neg.size > 0 and (got[neg] == 0).all() and not np.signbit(got[neg]).any()
    full = np.zeros(nd, bool)
    full[np.unique(dst)] = True
    assert np.abs(got - want)[full].max() < 1e-3


@pytest.mark.parametrize('bad', ['past_end', 'far_past_end', 'negative'])
def test_out_of_range_destination_raises(bad):
    """An out-of-range dst raises on an untrusted call, also where it follows a run of num_dst - 1 in its warp."""
    lib = _lib()
    rng = np.random.default_rng(3)
    nd, c_in, d = 700, 32, 300
    dst = np.sort(rng.integers(0, nd, EDGES)).astype(np.int32)
    i = 128 * 1000 + 40                                        # inside the tile of rows 128000 .. 128127
    if bad == 'past_end':
        dst[128 * 1000:i] = nd - 1
        dst[i] = nd
    else:
        dst[i] = nd + 1000 if bad == 'far_past_end' else -1
    src = rng.integers(0, nd, EDGES).astype(np.int32)
    f = _cuda((rng.standard_normal((nd, c_in)) * 0.5).astype(np.float32))
    x = _cuda((rng.standard_normal((nd, 3)) * 20).astype(np.float32))
    layer = _gnn_layer(lib, c_in, d, *_gnn_weights(rng, c_in, d))
    with pytest.raises(lib.PointGNNError):
        layer.edge_mlp_max(f, x, x, None, _cuda(src), _cuda(dst), nd)
    dst[i] = nd - 1
    good = layer.edge_mlp_max(f, x, x, None, _cuda(src), _cuda(np.sort(dst)), nd)
    assert (good > FMIN).any()

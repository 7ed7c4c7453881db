"""The tensor-core kernel (wg_gemm_kernel) at sizes where every CTA runs many tiles: the W ring then wraps through
both barrier parities many times and across tile boundaries, and the producer warpgroup runs far ahead of the
consumers.  Every instruction shape (64x1, 128x1, 96x2, 128x2, 152x2) and every producer / epilogue pair is covered,
against NumPy fp32."""
import numpy as np
import pytest
import torch

from oracle import gnn as ognn

pytestmark = pytest.mark.gpu
EDGES = 400000      # > 20 tiles of 128 rows per CTA on 132 SMs


def _need_tc():
    from pointgnn_b200 import _lib
    if not _lib.tc_available():
        pytest.skip('tensor-core path needs an sm_90 device')


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _mixed_dst(rng, e, nd):
    # half the edges spread over all destinations, half on four long segments spanning many tiles
    return np.sort(np.concatenate([rng.integers(0, nd, e // 2), rng.integers(10, 14, e - e // 2)]))


@pytest.mark.parametrize('n', [64, 128, 192, 256, 300, 600])
def test_dense_many_tiles_per_cta(n):
    """ROWS producer + store epilogue: 60 000 rows (469 tiles), bias / ReLU / residual; 600 wide runs as two 152x2
    column blocks, the others as one launch of the instruction shape N pads to."""
    _need_tc()
    from pointgnn_b200 import _lib
    rng = np.random.default_rng(n)
    m, k = 60000, 300
    x = rng.standard_normal((m, k)).astype(np.float32)
    w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
    b = rng.standard_normal(n).astype(np.float32)
    r = rng.standard_normal((m, n)).astype(np.float32)
    for relu in (True, False):
        for res in (None, r):
            want = x @ w + b
            if relu:
                want = np.maximum(want, 0)
            if res is not None:
                want = want + res
            before = _lib.tc_launch_count(1)
            got = _lib.fully_connected(_cuda(x), _cuda(w), _cuda(b), relu, residual=None if res is None else _cuda(res),
                                       precision=1).cpu().numpy()
            assert _lib.tc_launch_count(1) - before == (2 if n > 304 else 1), n
            assert got.shape == want.shape and np.abs(got - want).max() < 3e-4, (n, relu, res is None)


@pytest.mark.parametrize('d,c_in', [(300, 300), (256, 256), (64, 32), (128, 300)])
def test_gnn_edge_many_tiles_per_cta(d, c_in):
    """GNN producer + segment-max epilogue over 400 000 edges, against NumPy and the FFMA kernel's tolerance."""
    _need_tc()
    from pointgnn_b200 import _lib
    rng = np.random.default_rng(d + c_in)
    nv = 700
    dst = _mixed_dst(rng, EDGES, nv)
    src = rng.integers(0, nv, EDGES)
    f = (rng.standard_normal((nv, c_in)) * 0.5).astype(np.float32)
    x = (rng.standard_normal((nv, 3)) * 20).astype(np.float32)
    xd = x + (rng.standard_normal((nv, 3)) * 0.1).astype(np.float32)
    w1 = (rng.standard_normal((c_in + 3, d)) / np.sqrt(c_in)).astype(np.float32)
    b1 = (rng.standard_normal(d) * 0.1).astype(np.float32)
    w2 = (rng.standard_normal((d, d)) / np.sqrt(d)).astype(np.float32)
    b2 = (rng.standard_normal(d) * 0.1).astype(np.float32)
    e0 = np.concatenate([f[src], x[src] - xd[dst]], axis=1)
    want = ognn.graph_scatter_max_fn(np.maximum(np.maximum(e0 @ w1 + b1, 0) @ w2 + b2, 0), dst, nv)
    before = _lib.tc_launch_count(0)
    got = _lib.edge_mlp_max(1, _cuda(f), _cuda(x), _cuda(xd), None, _cuda(src.astype(np.int32)),
                            _cuda(dst.astype(np.int32)), nv, [_cuda(w1), _cuda(w2)], [_cuda(b1), _cuda(b2)],
                            precision=1).cpu().numpy()
    assert _lib.tc_launch_count(0) - before == 1, d
    empty = want == np.finfo(np.float32).min
    assert np.array_equal(got == np.finfo(np.float32).min, empty)
    assert np.abs(got - want)[~empty].max() < 1e-3, d


@pytest.mark.parametrize('dims', [(4, 32, 64, 128, 300), (4, 32, 64, 128, 256, 512), (4, 16, 64, 200),
                                  (4, 32, 128, 64)])
def test_pool_chain_many_tiles_per_cta(dims):
    """POOL producer + store, ROWS + store, ROWS + segment max over 400 000 edges with keypoint indirection."""
    _need_tc()
    from pointgnn_b200 import _lib
    rng = np.random.default_rng(sum(dims))
    nv, nk = 900, 400
    ws = [(rng.standard_normal((dims[i], dims[i + 1])) / np.sqrt(dims[i])).astype(np.float32) for i in range(len(dims) - 1)]
    bs = [(rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32) for i in range(len(dims) - 1)]
    dst = _mixed_dst(rng, EDGES, nk)
    src = rng.integers(0, nv, EDGES)
    f = rng.random((nv, 1)).astype(np.float32)
    x = (rng.standard_normal((nv, 3)) * 20).astype(np.float32)
    kp = rng.integers(0, nv, nk)
    h = np.concatenate([f[src], x[src] - x[kp[dst]]], axis=1)
    for w, b in zip(ws, bs):
        h = np.maximum(h @ w + b, 0)
    want = ognn.graph_scatter_max_fn(h, dst, nk)
    before = _lib.tc_launch_count(0)
    got = _lib.edge_mlp_max(0, _cuda(f), _cuda(x), _cuda(x), _cuda(kp.astype(np.int32)), _cuda(src.astype(np.int32)),
                            _cuda(dst.astype(np.int32)), nk, [_cuda(w) for w in ws], [_cuda(b) for b in bs],
                            precision=1).cpu().numpy()
    assert _lib.tc_launch_count(0) - before == -(-dims[-1] // 304), dims
    empty = want == np.finfo(np.float32).min
    assert np.array_equal(got == np.finfo(np.float32).min, empty)
    scale = max(1.0, float(np.abs(want[~empty]).max()))
    assert np.abs(got - want)[~empty].max() < 1e-3 * scale, dims

"""The GNN edge layer with W resident in shared memory (wg_gnn_body): a CTA per column group, three independent
warpgroups on 64-row tiles.  Shapes and edge counts the other GNN tests do not reach: the 96 x 2 instruction shape,
edge counts around the 64-row tile and the three warpgroups of a CTA, a hidden layer too wide for a resident group,
and repeated calls."""
import numpy as np
import pytest
import torch

from oracle import gnn as ognn

pytestmark = pytest.mark.gpu
FLT_MIN = np.finfo(np.float32).min


def _lib():
    from pointgnn_b200 import _lib
    if not _lib.tc_available():
        pytest.skip('tensor-core path needs an sm_90 device')
    return _lib


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _case(rng, e, nv, c_in, d1, n):
    """e edges grouped by destination (long runs and single edges), GNN edge MLP [c_in + 3, d1, n]."""
    dst = np.sort(np.concatenate([rng.integers(0, nv, e // 2), rng.integers(3, 5, e - e // 2)]))
    src = rng.integers(0, nv, e)
    f = (rng.standard_normal((nv, c_in)) * 0.5).astype(np.float32)
    x = (rng.standard_normal((nv, 3)) * 20).astype(np.float32)
    xd = x + (rng.standard_normal((nv, 3)) * 0.1).astype(np.float32)
    w1 = (rng.standard_normal((c_in + 3, d1)) / np.sqrt(c_in)).astype(np.float32)
    b1 = (rng.standard_normal(d1) * 0.1).astype(np.float32)
    w2 = (rng.standard_normal((d1, n)) / np.sqrt(d1)).astype(np.float32)
    b2 = (rng.standard_normal(n) * 0.1).astype(np.float32)
    e0 = np.concatenate([f[src], x[src] - xd[dst]], axis=1)
    want = ognn.graph_scatter_max_fn(np.maximum(np.maximum(e0 @ w1 + b1, 0) @ w2 + b2, 0), dst, nv)
    args = (_cuda(f), _cuda(x), _cuda(xd), None, _cuda(src.astype(np.int32)), _cuda(dst.astype(np.int32)), nv,
            [_cuda(w1), _cuda(w2)], [_cuda(b1), _cuda(b2)])
    return args, want


def _run(lib, args, launches, **kw):
    before = lib.tc_launch_count(0)
    got = lib.edge_mlp_max(1, *args, precision=1, **kw).cpu().numpy()
    assert lib.tc_launch_count(0) - before == launches
    return got


def _close(got, want, what):
    empty = want == FLT_MIN
    assert np.array_equal(got == FLT_MIN, empty), what
    assert np.abs(got - want)[~empty].max() < 1e-3, what


@pytest.mark.parametrize('d', [160, 192])
def test_gnn_96x2(d):
    """Padded widths 160 and 192 run the 96 x 2 instance: two column groups of 96."""
    lib = _lib()
    rng = np.random.default_rng(d)
    args, want = _case(rng, 20000, 500, 64, d, d)
    _close(_run(lib, args, 1), want, d)


@pytest.mark.parametrize('e', [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 5000])
def test_gnn_edge_counts_around_tiles(e):
    """Up to 128 edges a CTA has fewer tiles than warpgroups; 192 fill one CTA slot exactly; 193 start the next."""
    lib = _lib()
    rng = np.random.default_rng(e)
    args, want = _case(rng, e, 300, 32, 300, 300)
    _close(_run(lib, args, 1), want, e)


def test_gnn_hidden_layer_too_wide_for_a_resident_group():
    """A 512-wide hidden layer: a 152-column group of W2 (kp = 512) needs 304 KB, so the layer runs as 64-wide
    column blocks, 5 launches for 300 outputs (each group 128 KB)."""
    lib = _lib()
    rng = np.random.default_rng(512)
    args, want = _case(rng, 30000, 600, 48, 512, 300)
    _close(_run(lib, args, 5), want, 'd1 = 512')


@pytest.mark.parametrize('activation', ['ReLU', 'ELU'])
def test_gnn_repeated_calls_bitwise_equal(activation):
    """The max is exact and the flush order does not matter: repeated calls agree bit for bit."""
    lib = _lib()
    from pointgnn_b200.models import gnn
    code = gnn.activation_fn_dict[activation]
    rng = np.random.default_rng(3)
    args, _ = _case(rng, 200000, 2000, 300, 300, 300)
    first = _run(lib, args, 1, activation=code)
    for _ in range(2):
        assert np.array_equal(_run(lib, args, 1, activation=code), first), activation

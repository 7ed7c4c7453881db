"""The segment max of a warp whose 16 rows hold two destinations (those of rows 0 and 15): each is reduce-scattered in
its own pass with the other's rows masked.  Checked against NumPy fp32 (BF16x3) and the FP16 oracle, and bit for bit
between the list as built and a permutation of it, at the instruction shapes 152 x 2 (n = 300), 128 x 2 (256) and
64 x 1, with ReLU and with Tanh (raw maxima through the sign-aware atomic), for the GNN edge layer (and the pooling
chain, whose two accumulator groups keep the segmented scan, on the same patterns): run boundaries at every row of a warp, two destinations interleaved row by row (not grouped), a last warp
whose rows 9 .. 15 are past the end of the list, and negative maxima."""
import numpy as np
import pytest
import torch

from oracle import gnn as ognn

pytestmark = pytest.mark.gpu
FMIN = np.finfo(np.float32).min
BF16X3, FP16 = 1, 2
CONFIGS = [(300, BF16X3, 'ReLU'), (300, FP16, 'Tanh'), (256, BF16X3, 'Tanh'), (256, FP16, 'ReLU'),
           (64, BF16X3, 'Tanh'), (64, FP16, 'ReLU')]
C_IN = 32


def _lib():
    from pointgnn_b200 import _lib
    if not _lib.tc_available():
        pytest.skip('tensor-core path needs an sm_90 device')
    return _lib


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _act(name, x):
    return np.maximum(x, 0) if name == 'ReLU' else np.tanh(x)


def _want(f, x, src, dst, nd, ws, bs, prec, act):
    if prec == FP16:
        return ognn.gnn_edge_layer(f, x, x, src, dst, nd, ws, bs, act=act, fp16=True)
    out = np.full((nd, ws[1].shape[1]), FMIN, np.float32)
    e0 = np.concatenate([f[src], x[src] - x[dst]], axis=1)
    np.maximum.at(out, dst, _act(act, _act(act, e0 @ ws[0] + bs[0]) @ ws[1] + bs[1]).astype(np.float32))
    return out


def _pattern(name):
    """(dst, num_dst)."""
    if name == 'boundaries':      # destination k has k % 17 + 1 edges: a run boundary at every row of a warp
        dst = np.repeat(np.arange(2000), np.arange(2000) % 17 + 1)
        return dst, 2000
    if name == 'interleaved':     # within each 16-row unit, two destinations alternate row by row
        u = np.arange(1500)
        dst = np.stack([2 * u, 2 * u + 1] * 8, axis=1).reshape(-1)
        return dst, 3000
    if name == 'tail':            # 16 k + 9 rows: the last unit's rows 9 .. 15 are past the end
        return np.repeat(np.arange(700), 23)[:16 * 900 + 9], 700
    raise ValueError(name)


@pytest.mark.parametrize('n,prec,act', CONFIGS)
@pytest.mark.parametrize('name', ['boundaries', 'interleaved', 'tail'])
def test_gnn_two_destination_warps(name, n, prec, act):
    from pointgnn_b200.models import gnn
    lib = _lib()
    rng = np.random.default_rng(sum(map(ord, name)) * 1000 + n * 10 + prec)
    dst, nd = _pattern(name)
    nv = max(nd, 500)
    src = rng.integers(0, nv, dst.size)
    f = (rng.standard_normal((nv, C_IN)) * 0.5).astype(np.float32)
    x = (rng.standard_normal((nv, 3)) * 3).astype(np.float32)
    ws = [(rng.standard_normal((C_IN + 3, n)) / np.sqrt(C_IN + 3)).astype(np.float32),
          (rng.standard_normal((n, n)) / np.sqrt(n)).astype(np.float32)]
    # the second layer's bias pushes most Tanh outputs below zero: negative maxima go through the sign-aware atomic
    bs = [(rng.standard_normal(n) * 0.1).astype(np.float32),
          (rng.standard_normal(n) * 0.1 - (3.0 if act == 'Tanh' else 0.0)).astype(np.float32)]
    layer = lib.PreparedLayer(lib.PG_LAYER_EDGE_GNN, [_cuda(w) for w in ws], [_cuda(b) for b in bs], [C_IN + 3, n, n],
                              prec, activation=gnn.activation_fn_dict[act])
    perm = rng.permutation(dst.size)
    outs = [layer.edge_mlp_max(_cuda(f), _cuda(x), _cuda(x), None, _cuda(s.astype(np.int32)),
                               _cuda(t.astype(np.int32)), nd) for s, t in ((src, dst), (src[perm], dst[perm]))]
    assert torch.equal(outs[0], outs[1]), 'the edge order changed a bit'
    got = outs[0].cpu().numpy()
    want = _want(f, x, src, dst, nd, ws, bs, prec, act)
    empty = want == FMIN
    assert np.array_equal(got == FMIN, empty)
    if act == 'Tanh':
        assert (got[~empty] < 0).mean() > 0.5
    scale = max(1.0, float(np.abs(want[~empty]).max()))
    assert float(np.abs(got - want)[~empty].max()) <= 1e-3 * scale


@pytest.mark.parametrize('dims', [(4, 32, 64, 128, 300), (4, 32, 64, 128, 256, 512)])
@pytest.mark.parametrize('name', ['boundaries', 'interleaved'])
def test_pool_two_destination_warps(name, dims):
    """The pooling chain (car dims; ped's 512 as <ROWS, SEGMAX> column blocks): the list as built and permuted agree
    bit for bit, and match the fp32 pooling kernel."""
    lib = _lib()
    rng = np.random.default_rng(sum(dims) + len(name))
    dst, nk = _pattern(name)
    nv = 5000
    ws = [_cuda((rng.standard_normal((dims[i], dims[i + 1])) / np.sqrt(dims[i])).astype(np.float32))
          for i in range(len(dims) - 1)]
    bs = [_cuda((rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32)) for i in range(len(dims) - 1)]
    src = rng.integers(0, nv, dst.size)
    f = _cuda(rng.random((nv, 1)).astype(np.float32))
    x = _cuda((rng.standard_normal((nv, 3)) * 20).astype(np.float32))
    kp = _cuda(rng.integers(0, nv, nk).astype(np.int32))
    layer = lib.PreparedLayer(lib.PG_LAYER_EDGE_POOL, ws, bs, list(dims), BF16X3)
    perm = rng.permutation(dst.size)
    outs = [layer.edge_mlp_max(f, x, x, kp, _cuda(s.astype(np.int32)), _cuda(t.astype(np.int32)), nk)
            for s, t in ((src, dst), (src[perm], dst[perm]))]
    assert torch.equal(outs[0], outs[1])
    want = lib.PreparedLayer(lib.PG_LAYER_EDGE_POOL, ws, bs, list(dims), 0).edge_mlp_max(
        f, x, x, kp, _cuda(src.astype(np.int32)), _cuda(dst.astype(np.int32)), nk)
    assert torch.equal(outs[0] == FMIN, want == FMIN)
    full = want > FMIN
    scale = max(1.0, float(want[full].abs().max()))
    assert float((outs[0] - want)[full].abs().max()) <= 1e-3 * scale

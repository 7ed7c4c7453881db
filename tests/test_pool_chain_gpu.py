"""The point-set pooling MLP as one on-chip chain: layer 0 in fp32, every following layer on the tensor cores with its
activations kept in shared memory, and the last one ending in the segment max.  Launch counts of the car and ped
shapes, and shapes at the shared-memory and ring boundaries against the NumPy chain."""
import numpy as np
import pytest
import torch

from oracle import gnn as ognn

pytestmark = pytest.mark.gpu
FLT_MIN = np.finfo(np.float32).min


@pytest.fixture(scope='module')
def lib():
    from pointgnn_b200 import _lib
    if not _lib.tc_available():
        pytest.skip('tensor-core path needs an sm_90 device')
    return _lib


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _pool_case(dims, e, pattern, seed, nv=900, nk=400):
    """Random weights, points and a destination-sorted edge list, and the NumPy segment max of the MLP."""
    rng = np.random.default_rng(seed)
    ws = [(rng.standard_normal((dims[i], dims[i + 1])) / np.sqrt(dims[i])).astype(np.float32)
          for i in range(len(dims) - 1)]
    bs = [(rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32) for i in range(len(dims) - 1)]
    if pattern == 'long':
        dst = np.sort(rng.integers(0, 3, e))                  # segments spanning many tiles
    elif pattern == 'short':
        dst = np.sort(rng.integers(0, nk, e))                 # about one edge per segment, many empty
    else:
        dst = np.sort(np.concatenate([rng.integers(0, nk, e // 2), rng.integers(10, 14, e - e // 2)]))
    src = rng.integers(0, nv, e)
    f = rng.random((nv, 1)).astype(np.float32)
    x = (rng.standard_normal((nv, 3)) * 20).astype(np.float32)
    kp = rng.integers(0, nv, nk)
    h = np.concatenate([f[src], x[src] - x[kp[dst]]], axis=1)
    for w, b in zip(ws, bs):
        h = np.maximum(h @ w + b, 0)
    want = ognn.graph_scatter_max_fn(h, dst, nk)
    args = (_cuda(f), _cuda(x), _cuda(x), _cuda(kp.astype(np.int32)), _cuda(src.astype(np.int32)),
            _cuda(dst.astype(np.int32)), nk, [_cuda(w) for w in ws], [_cuda(b) for b in bs])
    return args, want


def _run_counted(lib, args):
    """One tensor-core pooling call and its (segment-max, dense) tensor-core launches."""
    before = (lib.tc_launch_count(0), lib.tc_launch_count(1))
    got = lib.edge_mlp_max(0, *args, precision=1).cpu().numpy()
    return got, (lib.tc_launch_count(0) - before[0], lib.tc_launch_count(1) - before[1])


def _check(got, want, what):
    empty = want == FLT_MIN
    assert np.array_equal(got == FLT_MIN, empty), what
    if (~empty).any():
        scale = max(1.0, float(np.abs(want[~empty]).max()))
        err = float(np.abs(got - want)[~empty].max())
        assert err < 1e-3 * scale, (what, err, scale)


def test_car_pooling_is_one_launch(lib):
    """4 -> 32 -> 64 -> 128 -> 300: the whole MLP and the segment max in a single tensor-core launch."""
    args, want = _pool_case((4, 32, 64, 128, 300), 5000, 'mixed', 1)
    got, (seg, dense) = _run_counted(lib, args)
    assert (seg, dense) == (1, 0)
    _check(got, want, 'car')


def test_ped_pooling_stores_the_last_input_once(lib):
    """4 -> 32 -> 64 -> 128 -> 256 -> 512: the chain up to 256 stores its rows once, then the 512-wide last layer
    runs as two column blocks of the segment max."""
    args, want = _pool_case((4, 32, 64, 128, 256, 512), 5000, 'mixed', 2)
    got, (seg, dense) = _run_counted(lib, args)
    assert (seg, dense) == (2, 1)
    _check(got, want, 'ped')


@pytest.mark.parametrize('dims', [
    (4, 20, 200, 64),                 # intermediates padded up to an instruction width (20 -> 32 k, 200 -> 256 n)
    (4, 32, 304, 128),                # an intermediate of 304: the widest region, ring of two stages
    (4, 64, 256, 300),                # last input 256: four 304-wide stages next to 2 x 64 KB of regions
    (4, 64, 304, 300),                # last input 304: 2 x 76 KB of regions, two stages
    (4, 300, 304, 304, 304),          # every on-chip layer as wide as one launch
    (4, 16, 64, 304, 600),            # wide last layer: the chain stores a 304-wide input
    (4, 8, 12, 16, 20, 24, 28, 32, 64),   # the deepest edge MLP (8 layers): six chained layers
])
def test_chain_boundary_shapes(lib, dims):
    for case, (e, pattern) in enumerate(((1, 'short'), (257, 'long'), (5000, 'mixed'))):
        args, want = _pool_case(dims, e, pattern, sum(dims) + case)
        got, (seg, dense) = _run_counted(lib, args)
        wide = dims[-1] > 304
        assert (seg, dense) == ((2, 1) if wide else (1, 0)), (dims, case)
        _check(got, want, (dims, case))


@pytest.mark.parametrize('dims', [(4, 32, 64, 128, 300), (4, 64, 304, 300)])
def test_chain_many_tiles_per_cta(lib, dims):
    """Enough edges for several tiles per CTA: the W ring and the A regions carry over from tile to tile."""
    args, want = _pool_case(dims, 200000, 'short', 7, nv=5000, nk=20000)
    got, (seg, dense) = _run_counted(lib, args)
    assert (seg, dense) == (1, 0)
    _check(got, want, dims)

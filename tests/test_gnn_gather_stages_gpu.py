"""The GNN edge layer's staged P gather (GnnGather in pg_tc.cu): each warpgroup copies its rows of P into shared
memory a 16-k chunk ahead of its wgmmas, and the copies run on from a tile's last chunk into the warpgroup's next tile.
Hidden layers of one chunk (every copy crosses into the next tile) and more; edge counts where warpgroups run no tile,
one tile and several; destination runs across tile boundaries; hidden widths on both sides of the shared-memory fit
limits; repeated calls."""
import numpy as np
import pytest
import torch

from oracle import gnn as ognn

pytestmark = pytest.mark.gpu
FLT_MIN = np.finfo(np.float32).min
# 132 SMs, two column groups of a 300-wide layer: 66 CTA slots of three warpgroups, 64-row tiles
ONE_TILE_EACH = 198 * 64


def _lib():
    from pointgnn_b200 import _lib
    if not _lib.tc_available():
        pytest.skip('tensor-core path needs an sm_90 device')
    return _lib


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _act(name, x):
    return np.maximum(x, 0) if name == 'ReLU' else np.where(x > 0, x, np.expm1(np.minimum(x, 0)))


def _case(rng, dst, nv, c_in, d1, n, act='ReLU'):
    """Edges grouped by destination dst (sorted), GNN edge MLP [c_in + 3, d1, n] with activation act."""
    e = len(dst)
    src = rng.integers(0, nv, e)
    f = (rng.standard_normal((nv, c_in)) * 0.5).astype(np.float32)
    x = (rng.standard_normal((nv, 3)) * 20).astype(np.float32)
    xd = x + (rng.standard_normal((nv, 3)) * 0.1).astype(np.float32)
    w1 = (rng.standard_normal((c_in + 3, d1)) / np.sqrt(c_in)).astype(np.float32)
    b1 = (rng.standard_normal(d1) * 0.1).astype(np.float32)
    w2 = (rng.standard_normal((d1, n)) / np.sqrt(d1)).astype(np.float32)
    b2 = (rng.standard_normal(n) * 0.1).astype(np.float32)
    e0 = np.concatenate([f[src], x[src] - xd[dst]], axis=1).astype(np.float64)
    want = ognn.graph_scatter_max_fn(_act(act, _act(act, e0 @ w1 + b1) @ w2 + b2).astype(np.float32), dst, nv)
    args = (_cuda(f), _cuda(x), _cuda(xd), None, _cuda(src.astype(np.int32)), _cuda(dst.astype(np.int32)), nv,
            [_cuda(w1), _cuda(w2)], [_cuda(b1), _cuda(b2)])
    return args, want


def _random_dst(rng, e, nv):
    """Long runs and single edges."""
    return np.sort(np.concatenate([rng.integers(0, nv, e // 2), rng.integers(3, 5, e - e // 2)]))


def _run(lib, args, launches, act='ReLU'):
    from pointgnn_b200.models import gnn
    before = lib.tc_launch_count(0)
    got = lib.edge_mlp_max(1, *args, precision=1, activation=gnn.activation_fn_dict[act]).cpu().numpy()
    assert lib.tc_launch_count(0) - before == launches
    return got


def _close(got, want, what):
    empty = want == FLT_MIN
    assert np.array_equal(got == FLT_MIN, empty), what
    assert np.abs(got - want)[~empty].max() < 1e-3, what


@pytest.mark.parametrize('act', ['ReLU', 'ELU'])
@pytest.mark.parametrize('d1', [16, 32, 48, 64])
def test_gnn_chunks_per_tile(d1, act):
    """1, 2, 3 and 4 chunks of 16 k; every warpgroup takes several tiles."""
    lib = _lib()
    rng = np.random.default_rng(d1)
    args, want = _case(rng, _random_dst(rng, 4 * ONE_TILE_EACH + 777, 3000), 3000, 32, d1, 300, act)
    _close(_run(lib, args, 1, act), want, (d1, act))


@pytest.mark.parametrize('e', [100 * 64, ONE_TILE_EACH, ONE_TILE_EACH + 1, 2 * ONE_TILE_EACH - 5, 40000])
def test_gnn_tiles_per_warpgroup(e):
    """Some warpgroups without a tile, every one with exactly one, a few with two, then several each."""
    lib = _lib()
    rng = np.random.default_rng(e)
    args, want = _case(rng, _random_dst(rng, e, 2000), 2000, 64, 300, 300)
    _close(_run(lib, args, 1), want, e)


@pytest.mark.parametrize('run', [1, 7, 60, 64, 65, 100, 193])
def test_gnn_destination_runs_across_tiles(run):
    """Runs of equal destinations that straddle 64-row tile boundaries, and the tiles of one warpgroup."""
    lib = _lib()
    rng = np.random.default_rng(run)
    e = 3 * ONE_TILE_EACH + 11
    nv = e // run + 1
    args, want = _case(rng, np.arange(e) // run, nv, 32, 128, 300)
    _close(_run(lib, args, 1), want, run)


@pytest.mark.parametrize('d1,c_in,n,launches', [
    (352, 32, 300, 1),   # 152-column group: 352 x 152 x 4 B of W + 12 KB of stages fit in 227 KB
    (368, 32, 300, 5),   # no longer: five 64-wide column blocks
    (848, 16, 32, 1),    # 64-column group: the deepest that fits
    (864, 16, 32, 0),    # the fp32 edge kernel
])
def test_gnn_hidden_width_at_the_fit_limits(d1, c_in, n, launches):
    lib = _lib()
    rng = np.random.default_rng(d1)
    args, want = _case(rng, _random_dst(rng, 20000, 800), 800, c_in, d1, n)
    _close(_run(lib, args, launches), want, d1)


@pytest.mark.parametrize('act', ['ReLU', 'ELU'])
def test_gnn_staged_gather_repeated_calls_bitwise_equal(act):
    lib = _lib()
    rng = np.random.default_rng(5)
    args, _ = _case(rng, _random_dst(rng, 150000, 2000), 2000, 48, 48, 300, act)
    first = _run(lib, args, 1, act)
    for _ in range(2):
        assert np.array_equal(_run(lib, args, 1, act), first), act

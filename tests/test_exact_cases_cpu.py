"""The integer edge-layer and dense cases of test_exact_edge_gpu.py, proved right without a GPU: the exactness
conditions of oracle/synth.py hold (the worst margins are printed), the float64 oracle, the float32 oracle and the
FP16 oracle agree exactly after the cast to float32 (so no routing or arithmetic of the library can differ on these
inputs), deleting one edge changes the expected sum and mean, and the edge lists have the structure they claim."""
import numpy as np
import pytest

from oracle import synth

GNN_DIMS = [(35, 300, 300), (35, 256, 256), (35, 192, 192), (35, 64, 64), (35, 512, 300)]
CAR = (4, 32, 64, 128, 300)
PED = (4, 32, 64, 128, 256, 512)
# a pooling chain whose last layer is wider than one launch (as PED's 256 -> 512): its input is stored per edge, in
# slices of 2^20 rows.  Narrow before the split, so that the 1.3 M-edge list stays cheap on the CPU
SPLIT = (4, 16, 16, 16, 320)
TAILS = ['tail_%d' % e for e in synth.TAIL_SIZES]

# (layer, dims, edge list, activations): every pairing test_exact_edge_gpu.py runs.  The slice lists carry a
# destination of degree > 2^18, whose sum bounds the per-edge values: only narrow layers fit EXACT_SUM there, and a
# narrow hidden layer keeps them cheap (n = 192 still runs as two 96-column groups)
EDGE_CASES = (
    [('gnn', d, lst, ('ReLU', 'ReLU6')) for d in GNN_DIMS for lst in ['mixed', 'tails']]
    + [('gnn', (35, 64, 64), 'slices', ('ReLU', 'ReLU6')), ('gnn', (35, 32, 192), 'slices', ('ReLU',))]
    + [('pool', d, lst, ('ReLU', 'ReLU6', 'NONE')) for d in (CAR, PED) for lst in ['mixed', 'tails']]
    + [('pool', SPLIT, 'pool_slices', ('ReLU',))]
)

# dense: m = 60 000 rows (a partial last tile), k in {35, 300}, n in {7, 300, 600} (600: two column blocks)
DENSE_M = 60000
DENSE_SHAPES = [(k, n) for k in (35, 300) for n in (7, 300, 600)]


def case_id(layer, dims, lst):
    return '%s%s-%s' % (layer, 'x'.join(map(str, dims)), lst)


_lists = {}
_cases = {}


def edge_list(name):
    if name not in _lists:
        _lists[name] = synth.exact_edge_list(name)
    return _lists[name]


def lists_of(lst):
    """The edge lists a case table entry names ('tails': all of TAILS)."""
    return TAILS if lst == 'tails' else [lst]


def edge_case(layer, dims, name):
    """The integer layer on the vertices of edge list `name` (one seed per layer shape)."""
    key = (layer, tuple(dims), name)
    if key not in _cases:
        _cases[key] = synth.exact_edge_case(layer, dims, edge_list(name)['num_dst'], seed=sum(dims) + len(dims))
    return _cases[key]


def dense_case(k, n, residual):
    return synth.exact_dense_case(DENSE_M, (k, n), seed=k * 1000 + n, residual=residual)


def _worst(m):
    return max(m['value'], m['dot'], m['sum'])


# ---- the exactness conditions and the oracles ------------------------------------------------------------------------
@pytest.mark.parametrize('layer,dims,lst,acts', EDGE_CASES, ids=[case_id(*c[:3]) for c in EDGE_CASES])
def test_edge_case_is_exact(layer, dims, lst, acts):
    for name in lists_of(lst):
        edges = edge_list(name)
        case = edge_case(layer, dims, name)
        for act in acts:
            m = synth.exact_margins(case, edges, act)
            print('%s %s: value %.4f dot %.2e sum %.4f' % (case_id(layer, dims, name), act, m['value'], m['dot'],
                                                            m['sum']))
            assert m['integer'] and m['weights'], m
            assert _worst(m) < 1.0, m
            want = synth.exact_edge_reference(case, edges, act, 'sum')
            assert np.array_equal(synth.exact_edge_reference(case, edges, act, 'sum', dtype=np.float32), want)
            assert np.array_equal(synth.exact_edge_reference(case, edges, act, 'sum', dtype=np.float32, fp16=True),
                                  want)


def _run_of(edges, d):
    """The edges of destination d as their own list (the sum and the mean of d depend on nothing else)."""
    keep = edges['dst'] == d
    return dict(src=edges['src'][keep], dst=edges['dst'][keep], num_dst=edges['num_dst'])


@pytest.mark.parametrize('layer,dims,lst,acts', [c for c in EDGE_CASES if c[2] in ('mixed', 'tails')],
                         ids=[case_id(*c[:3]) for c in EDGE_CASES if c[2] in ('mixed', 'tails')])
def test_deleting_an_edge_changes_the_sum_and_the_mean(layer, dims, lst, acts):
    rng = np.random.default_rng(sum(dims))
    for name in lists_of(lst):
        edges = edge_list(name)
        case = edge_case(layer, dims, name)
        for e in rng.choice(len(edges['src']), min(3, len(edges['src'])), replace=False):
            d = int(edges['dst'][e])
            run = _run_of(edges, d)
            pos = int(np.flatnonzero(run['src'] == edges['src'][e])[0])
            less = dict(run, src=np.delete(run['src'], pos), dst=np.delete(run['dst'], pos))
            for act in acts:
                for agg in ('sum', 'mean'):
                    a = synth.exact_edge_reference(case, run, act, agg)[d]
                    b = synth.exact_edge_reference(case, less, act, agg)[d]
                    if agg == 'sum':
                        assert (a != b).any(), (name, e, act)
                        # under ReLU and ReLU6 every edge adds >= 1 to every column
                        assert act == 'NONE' or (a - b >= 1).all(), (name, e, act)
                    elif act != 'ReLU6':
                        # ReLU6 saturates: two edges of a run may give the same row, and dropping one of them leaves
                        # the mean as it was.  The kernels count a destination's edges apart from the MLP, so an edge
                        # the MLP dropped still changes the mean through the sum
                        assert (a != b).any(), (name, e, act)


@pytest.mark.parametrize('residual', [False, True])
@pytest.mark.parametrize('k,n', DENSE_SHAPES)
def test_dense_case_is_exact(k, n, residual):
    case = dense_case(k, n, residual)
    for act in ('ReLU', 'NONE'):
        m = synth.exact_dense_margins(case, [act])
        print('dense %dx%d residual %s %s: value %.4f dot %.2e' % (k, n, residual, act, m['value'], m['dot']))
        assert m['integer'] and m['weights'] and _worst(m) < 1.0, m
        want = synth.exact_dense_reference(case, [act])
        assert np.array_equal(synth.exact_dense_reference(case, [act], dtype=np.float32), want)
        assert np.array_equal(synth.exact_dense_reference(case, [act], dtype=np.float32, fp16=True), want)


# ---- the edge lists ----------------------------------------------------------------------------------------------------
def _starts(edges):
    d = edges['dst']
    return np.flatnonzero(np.concatenate([[True], d[1:] != d[:-1]])) if len(d) else np.zeros(0, np.int64)


def test_every_list_is_grouped_and_in_range():
    for name in ['mixed', 'slices', 'pool_slices'] + TAILS:
        e = edge_list(name)
        assert len(e['src']) == len(e['dst'])
        assert e['src'].dtype == np.int32 and e['dst'].dtype == np.int32
        assert (np.diff(e['dst']) >= 0).all(), name
        assert e['src'].min() >= 0 and e['src'].max() < e['num_dst'], name
        assert e['dst'].min() >= 0 and e['dst'].max() < e['num_dst'], name


def test_mixed_list():
    e = edge_list('mixed')
    E = len(e['dst'])
    assert 45000 <= E <= 65000 and E % 16 != 0          # a partial last unit
    deg = np.bincount(e['dst'], minlength=e['num_dst'])
    assert deg[e['marks']['hub']] == 3000
    assert np.sort(deg)[-2] <= 40 and deg.min() == 0
    assert (deg[e['marks']['empty']] == 0).all()
    assert deg[-1] == 0 and e['dst'].max() < e['num_dst'] - 1          # empty destinations past the last edge
    middle = np.flatnonzero(deg[:e['dst'].max()] == 0)
    assert len(middle) >= 3                                             # and between edges
    starts = _starts(e)
    assert set(starts % 64) == set(range(64)) and set(starts % 16) == set(range(16))


def test_slices_list():
    S = synth.ORDERED_SLICE
    e = edge_list('slices')
    E = len(e['dst'])
    assert E == 3 * S + 1000
    deg = np.bincount(e['dst'], minlength=e['num_dst'])
    big = e['marks']['big']
    rows = np.flatnonzero(e['dst'] == big)
    first, last = int(rows[0]), int(rows[-1])
    assert deg[big] > S
    assert first < S and last >= 2 * S                                  # covers the second slice and both boundaries
    assert first % 16 and (last + 1) % 16                               # starts and ends mid-unit
    ends = e['marks']['ends_at_slice']
    assert np.flatnonzero(e['dst'] == ends)[-1] == 3 * S - 1
    single = np.flatnonzero(e['dst'] == e['marks']['single'])
    assert len(single) == 1 and single[0] == 3 * S
    assert deg[-1] == 0


def test_pool_slices_list():
    P, S = synth.STORE_SLICE, synth.ORDERED_SLICE
    e = edge_list('pool_slices')
    assert len(e['dst']) == P + S + 5
    rows = np.flatnonzero(e['dst'] == e['marks']['straddle'])
    assert rows[0] < P <= rows[-1]
    assert rows[0] % 16 and (rows[-1] + 1) % 16
    # the store slices 2^20 and 2^18 + 5 make 4 + 2 ordered slices, one fix-up each
    assert sum(-(-min(P, len(e['dst']) - s) // S) for s in range(0, len(e['dst']), P)) == 6


def test_tail_lists():
    for name, size in zip(TAILS, synth.TAIL_SIZES):
        e = edge_list(name)
        assert len(e['dst']) == size
        assert np.bincount(e['dst'], minlength=e['num_dst'])[-1] == 0

"""The aggregations of the reference's table (gnn.py:106-119): graph_scatter_max_fn, graph_scatter_sum_fn and
graph_scatter_mean_fn, as the reduction of the fused edge layers.

The oracle (oracle/gnn.py) takes the aggregation as an argument of its edge layers and of ``predict``; the max, the
aggregation of every shipped config, is pinned by the goldens.  The GPU tests compare the kernels against it."""
import os
import re

import numpy as np
import pytest

from oracle import gnn as ognn
from oracle.gnn import AGGREGATIONS, graph_net_auto_center, point_set_pooling, segment_reduce

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_segment_reduce_vs_loops():
    """Sorted and unsorted ids, empty segments, E = 0."""
    rng = np.random.default_rng(1)
    for e, k, sort in ((2000, 50, True), (2000, 50, False), (0, 7, True)):
        ids = rng.integers(0, k, e)
        ids[ids == 3] = 4
        if sort:
            ids = np.sort(ids)
        x = rng.standard_normal((e, 5))
        want = {'max': np.full((k, 5), np.finfo(np.float64).min), 'sum': np.zeros((k, 5))}
        for i in range(e):
            want['max'][ids[i]] = np.maximum(want['max'][ids[i]], x[i])
            want['sum'][ids[i]] += x[i]
        want['mean'] = want['sum'] / np.maximum(np.bincount(ids, minlength=k), 1)[:, None]
        for agg in AGGREGATIONS:
            got = segment_reduce(x, ids, k, agg)
            assert np.allclose(got, want[agg], rtol=1e-12, atol=1e-12), (agg, e, sort)
        assert (segment_reduce(x, ids, k, 'sum')[3] == 0).all() and (segment_reduce(x, ids, k, 'mean')[3] == 0).all()


def _mlp64(h, ws, bs, last_linear=False):
    for i, (w, b) in enumerate(zip(ws, bs)):
        h = h @ w.astype(np.float64) + b.astype(np.float64)
        if not (last_linear and i == len(ws) - 1):
            h = np.maximum(h, 0)
    return h


def _scope_weights(w, scope, n):
    names = [scope + '/fully_connected' + ('' if i == 0 else '_%d' % i) for i in range(n)]
    return [w[n + '/weights'] for n in names], [w[n + '/biases'] for n in names]


@pytest.mark.parametrize('aggregation', ['sum', 'mean'])
def test_oracle_layers_vs_numpy(aggregation, car):
    """The oracle's pooling and GNN layers with a sum or a mean, in float64, against the composition written out."""
    coords, keypoints, edges = car.graph_tuple()
    w = car.weights
    # pooling layer1 on the level-0 graph
    lc = car.layer_configs[0]
    feats, xyz, kp, ed = car.graph['intensity'].astype(np.float64), coords[0].astype(np.float64), keypoints[0], edges[0]
    got = point_set_pooling(w, 'layer1', feats, xyz, kp, ed, aggregation=aggregation, chunk=10000, **lc['kwargs'])
    src, dst = ed[:, 0], ed[:, 1]
    h = _mlp64(np.concatenate([feats[src], xyz[src] - xyz[kp[dst, 0]]], axis=1),
               *_scope_weights(w, 'layer1/extract_vertex_features', len(lc['kwargs']['point_MLP_depth_list'])))
    agg = np.zeros((len(kp), h.shape[1]))
    np.add.at(agg, dst, h)
    if aggregation == 'mean':
        agg /= np.maximum(np.bincount(dst, minlength=len(kp)), 1)[:, None]
    want = _mlp64(agg, *_scope_weights(w, 'layer1/combined_features', len(lc['kwargs']['output_MLP_depth_list'])))
    assert np.abs(got - want).max() <= 1e-9 * max(1.0, np.abs(want).max())
    # GNN layer3 (auto offset) on the level-1 graph
    lc = [c for c in car.layer_configs if c['scope'] == 'layer3'][0]
    kw = lc['kwargs']
    rng = np.random.default_rng(5)
    f = np.abs(rng.standard_normal((coords[1].shape[0], 300))) * 0.3
    x1, ed = coords[1].astype(np.float64), edges[1]
    got = graph_net_auto_center(w, 'layer3', f, x1, None, ed, aggregation=aggregation, chunk=50000, **kw)
    src, dst = ed[:, 0], ed[:, 1]
    off = x1 + _mlp64(f, *_scope_weights(w, 'layer3', len(kw['auto_offset_MLP_depth_list'])), last_linear=True)
    h = _mlp64(np.concatenate([f[src], x1[src] - off[dst]], axis=1),
               *_scope_weights(w, 'layer3/extract_vertex_features', len(kw['edge_MLP_depth_list'])))
    agg = np.zeros((len(f), h.shape[1]))
    np.add.at(agg, dst, h)
    if aggregation == 'mean':
        agg /= np.maximum(np.bincount(dst, minlength=len(f)), 1)[:, None]
    want = f + _mlp64(agg, *_scope_weights(w, 'layer3/combined_features', len(kw['update_MLP_depth_list'])),
                      last_linear=True)
    assert np.abs(got - want).max() <= 1e-9 * max(1.0, np.abs(want).max())


def test_oracle_with_max_reproduces_goldens(car):
    coords, keypoints, edges = car.graph_tuple()
    logits, boxes = ognn.predict(car.weights, car.layer_configs, car.config['num_classes'], 7, car.graph['intensity'],
                                 coords, keypoints, edges, aggregation='max')
    assert np.abs(logits - car.gnn['logits']).max() < 2e-5
    assert np.abs(boxes - car.gnn['boxes']).max() < 2e-5


def test_header_constants_equal_the_python_table():
    from pointgnn_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'pointgnn_b200.h')) as f:
        text = f.read()
    header = dict((k, int(v, 0)) for k, v in re.findall(r'#define PG_AGG_(\w+) (0x[0-9a-f]+|\d+)\b', text))
    assert header == {'MAX': 0, 'SUM': 1, 'MEAN': 2, 'SHIFT': 10, 'MASK': 0xc00}
    for macro, value in header.items():
        assert getattr(_lib, 'PG_AGG_' + macro) == value
    assert _lib.AGGREGATIONS == {'max': header['MAX'], 'sum': header['SUM'], 'mean': header['MEAN']}
    # the field does not overlap the precision, the trusted flag or the activation's bits
    for taken in (_lib.PG_PRECISION_MASK, _lib.PG_FLAG_TRUSTED_INDICES, _lib.PG_FLAG_ACTIVATION, _lib.PG_ACT_MASK):
        assert taken & _lib.PG_AGG_MASK == 0
    assert re.search(r'#define PG_AGGREGATION\(code\) \(\(code\) << PG_AGG_SHIFT\)', text)


def test_unknown_aggregation_name_raises_before_any_launch():
    """No tensor is touched: None arguments would fail on a launch."""
    from pointgnn_b200 import _lib
    for name in ('median', 'MAX', None, 0):
        with pytest.raises(_lib.PointGNNError, match='unknown aggregation'):
            _lib.edge_mlp_max(1, None, None, None, None, None, None, 10, [], [], aggregation=name)
        layer = object.__new__(_lib.PreparedLayer)
        with pytest.raises(_lib.PointGNNError, match='unknown aggregation'):
            layer.edge_mlp_max(None, None, None, None, None, None, 10, aggregation=name)


def test_fusable_accepts_the_package_plug_ins_by_identity():
    from pointgnn_b200.models import gnn

    def user_sum(*args):
        return gnn.graph_scatter_sum_fn(*args)

    for cls in (gnn.PointSetPooling, gnn.GraphNetAutoCenter):
        assert cls()._fusable('NONE') == 'max'
        assert cls(aggregation_fn=gnn.graph_scatter_sum_fn)._fusable('NONE') == 'sum'
        assert cls(aggregation_fn=gnn.graph_scatter_mean_fn)._fusable('NONE') == 'mean'
        assert cls(aggregation_fn=user_sum)._fusable('NONE') is None
        assert cls(aggregation_fn=gnn.graph_scatter_sum_fn)._fusable('BN') is None

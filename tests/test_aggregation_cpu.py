"""The aggregations of the reference's table (gnn.py:106-119): graph_scatter_max_fn, graph_scatter_sum_fn and
graph_scatter_mean_fn, as the reduction of the fused edge layers.

The CPU oracle package implements the max, the aggregation of every shipped config, and stays as it is: the goldens
pin it.  This module restates its two edge layers with any aggregation (``point_set_pooling``, ``graph_net_auto_center``)
and the FP16 oracle's edge layers the same way (``f16_pool_edge``, ``f16_gnn_edge``); ``aggregation_oracle()`` and
``f16_aggregation_oracle()`` run the whole-model oracles with them.  The GPU tests compare the kernels against these."""
import contextlib
import functools
import os
import re

import numpy as np
import pytest

import fp16_oracle as f16o
from oracle import gnn as ognn
from test_activations_cpu import activate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AGGREGATIONS = ('max', 'sum', 'mean')


def segment_reduce(x, dst, num, aggregation):
    """tf.math.unsorted_segment_max / _sum / _mean in x's dtype, dst in any order; an empty segment gives the lowest
    float (max) or 0 (sum, mean)."""
    dst = np.asarray(dst).reshape(-1).astype(np.int64)
    if aggregation == 'max':
        return ognn.graph_scatter_max_fn(x, dst, num)
    out = np.zeros((int(num), x.shape[1]), x.dtype)
    if len(dst):
        order = np.argsort(dst, kind='stable')
        d, xs = dst[order], x[order]
        starts = np.flatnonzero(np.concatenate([[True], d[1:] != d[:-1]]))
        out[d[starts]] = np.add.reduceat(xs, starts, axis=0)
    if aggregation == 'mean':
        out /= np.maximum(np.bincount(dst, minlength=int(num)), 1).astype(x.dtype)[:, None]
    return out


class _Reduction(object):
    """A segment reduction fed chunk by chunk: partial maxima or sums, the mean's division at the end."""

    def __init__(self, num, n, dtype, aggregation):
        self.aggregation = aggregation
        self.count = np.zeros(int(num), np.int64)
        self.out = segment_reduce(np.zeros((0, n), dtype), [], num, 'max' if aggregation == 'max' else 'sum')

    def add(self, x, dst):
        part = segment_reduce(x, dst, self.out.shape[0], 'max' if self.aggregation == 'max' else 'sum')
        if self.aggregation == 'max':
            np.maximum(self.out, part, out=self.out)
        else:
            self.out += part
        self.count += np.bincount(np.asarray(dst, np.int64), minlength=self.out.shape[0])

    def result(self):
        if self.aggregation == 'mean':
            self.out /= np.maximum(self.count, 1).astype(self.out.dtype)[:, None]
        return self.out


def _chunks(n, chunk):
    for s in range(0, n, chunk):
        yield s, min(n, s + chunk)


def point_set_pooling(weights, scope_name, point_features, point_coordinates, keypoint_indices, set_indices,
                      point_MLP_depth_list=None, point_MLP_normalization_type='NONE', point_MLP_activation_type='ReLU',
                      output_MLP_depth_list=None, output_MLP_normalization_type='NONE',
                      output_MLP_activation_type='ReLU', aggregation='max', chunk=1 << 16):
    """oracle.gnn.point_set_pooling (gnn.py:222-283) with the aggregation as an argument."""
    set_indices = np.asarray(set_indices).astype(np.int64)
    keypoint_indices = np.asarray(keypoint_indices).astype(np.int64)
    red = _Reduction(keypoint_indices.shape[0], point_MLP_depth_list[-1], point_features.dtype, aggregation)
    for s, e in _chunks(set_indices.shape[0], chunk):
        si = set_indices[s:e]
        kc = point_coordinates[keypoint_indices[si[:, 1]][:, 0]]
        x = np.concatenate([point_features[si[:, 0]], point_coordinates[si[:, 0]] - kc], axis=-1)
        sc = ognn._Scope(weights, scope_name).sub('extract_vertex_features')
        x = ognn.multi_layer_neural_network_fn(x, sc, Ks=point_MLP_depth_list, is_logits=False,
                                               normalization_type=point_MLP_normalization_type,
                                               activation_type=point_MLP_activation_type)
        red.add(x, si[:, 1])
    sc = ognn._Scope(weights, scope_name).sub('combined_features')
    return ognn.multi_layer_neural_network_fn(red.result(), sc, Ks=output_MLP_depth_list, is_logits=False,
                                              normalization_type=output_MLP_normalization_type,
                                              activation_type=output_MLP_activation_type)


def graph_net_auto_center(weights, scope_name, input_vertex_features, input_vertex_coordinates, NOT_USED, edges,
                          edge_MLP_depth_list=None, edge_MLP_normalization_type='NONE', edge_MLP_activation_type='ReLU',
                          update_MLP_depth_list=None, update_MLP_normalization_type='NONE',
                          update_MLP_activation_type='ReLU', auto_offset=False, auto_offset_MLP_depth_list=None,
                          auto_offset_MLP_normalization_type='NONE', auto_offset_MLP_feature_activation_type='ReLU',
                          aggregation='max', chunk=1 << 16):
    """oracle.gnn.graph_net_auto_center (gnn.py:298-373) with the aggregation as an argument."""
    edges = np.asarray(edges).astype(np.int64)
    coords = input_vertex_coordinates
    if auto_offset:
        coords = input_vertex_coordinates + ognn.multi_layer_neural_network_fn(
            input_vertex_features, ognn._Scope(weights, scope_name), Ks=auto_offset_MLP_depth_list, is_logits=True,
            normalization_type=auto_offset_MLP_normalization_type,
            activation_type=auto_offset_MLP_feature_activation_type)
    red = _Reduction(input_vertex_features.shape[0], edge_MLP_depth_list[-1], input_vertex_features.dtype, aggregation)
    for s, e in _chunks(edges.shape[0], chunk):
        ed = edges[s:e]
        x = np.concatenate([input_vertex_features[ed[:, 0]], input_vertex_coordinates[ed[:, 0]] - coords[ed[:, 1]]],
                           axis=-1)
        sc = ognn._Scope(weights, scope_name).sub('extract_vertex_features')
        x = ognn.multi_layer_neural_network_fn(x, sc, Ks=edge_MLP_depth_list, is_logits=False,
                                               normalization_type=edge_MLP_normalization_type,
                                               activation_type=edge_MLP_activation_type)
        red.add(x, ed[:, 1])
    sc = ognn._Scope(weights, scope_name).sub('combined_features')
    update = ognn.multi_layer_neural_network_fn(red.result(), sc, Ks=update_MLP_depth_list, is_logits=True,
                                                normalization_type=update_MLP_normalization_type,
                                                activation_type=update_MLP_activation_type)
    return update + input_vertex_features


@contextlib.contextmanager
def aggregation_oracle(aggregation):
    """The oracle package with both edge layers reducing by ``aggregation`` (predict looks them up at call time)."""
    saved = ognn.point_set_pooling, ognn.graph_net_auto_center
    ognn.point_set_pooling = functools.partial(point_set_pooling, aggregation=aggregation)
    ognn.graph_net_auto_center = functools.partial(graph_net_auto_center, aggregation=aggregation)
    try:
        yield ognn
    finally:
        ognn.point_set_pooling, ognn.graph_net_auto_center = saved


# ---- FP16 (precision code 2): rounds where the kernels round, as fp16_oracle does ----------------------------------
def f16_pool_edge(feat, xyz, kxyz, src, dst, num_dst, ws, bs, act='ReLU', aggregation='max', chunk=1 << 15):
    """fp16_oracle.pool_edge_max with the aggregation as an argument: every tensor-core layer's A operand is the
    previous layer's activation rounded once to FP16; bias, activation and the reduction stay fp32."""
    dims = [ws[0].shape[0]] + [w.shape[1] for w in ws]
    tc = f16o.pool_uses_tc(dims, act)
    red = _Reduction(num_dst, dims[-1], np.float32, aggregation)
    for s, e in _chunks(len(src), chunk):
        si, di = src[s:e], dst[s:e]
        x = np.concatenate([feat[si], xyz[si] - kxyz[di]], axis=1).astype(np.float32)
        for l, (w, b) in enumerate(zip(ws, bs)):
            y = f16o.tc_gemm(x, w) if tc and l > 0 else x @ w.astype(np.float32)
            x = activate(act, y + b.astype(np.float32)[None, :])
        red.add(x, di)
    return red.result()


def f16_gnn_edge(feat, xyz_src, xyz_dst, src, dst, num_dst, ws, bs, act='ReLU', aggregation='max', chunk=1 << 15):
    """fp16_oracle.gnn_edge_max with the aggregation as an argument: A = act(P[src] + (x_src - x_dst') @ W1[C:]) in
    fp32, rounded once to FP16; act(A @ W2 + b2) per edge in fp32, then the reduction."""
    dims = [ws[0].shape[0]] + [w.shape[1] for w in ws]
    c = feat.shape[1]
    tc = f16o.gnn_uses_tc(dims)
    if tc:
        p = f16o.fc(feat, ws[0][:c], bs[0], 'NONE')
    red = _Reduction(num_dst, dims[-1], np.float32, aggregation)
    for s, e in _chunks(len(src), chunk):
        si, di = src[s:e], dst[s:e]
        d = (xyz_src[si] - xyz_dst[di]).astype(np.float32)
        if tc:
            x = activate(act, p[si] + d @ ws[0][c:].astype(np.float32))
            x = activate(act, f16o.tc_gemm(x, ws[1]) + bs[1].astype(np.float32)[None, :])
        else:
            x = np.concatenate([feat[si], d], axis=1).astype(np.float32)
            for w, b in zip(ws, bs):
                x = activate(act, x @ w.astype(np.float32) + b.astype(np.float32)[None, :])
        red.add(x, di)
    return red.result()


@contextlib.contextmanager
def f16_aggregation_oracle(aggregation):
    """fp16_oracle with both edge layers reducing by ``aggregation`` (its layers look them up at call time)."""
    saved = f16o.pool_edge_max, f16o.gnn_edge_max
    f16o.pool_edge_max = functools.partial(f16_pool_edge, aggregation=aggregation)
    f16o.gnn_edge_max = functools.partial(f16_gnn_edge, aggregation=aggregation)
    try:
        yield f16o
    finally:
        f16o.pool_edge_max, f16o.gnn_edge_max = saved


# ---- tests ----------------------------------------------------------------------------------------------------------
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
    with aggregation_oracle('max') as o:
        logits, boxes = o.predict(car.weights, car.layer_configs, car.config['num_classes'], 7,
                                  car.graph['intensity'], coords, keypoints, edges)
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

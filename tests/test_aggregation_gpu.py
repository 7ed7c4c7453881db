"""The sum and the mean of the reference's aggregation table (gnn.py:111-119) through the fused edge layers: the GNN
edge layer, the car pooling chain and the ped pooling split (256 -> 512: a store launch, then the row launches), at
fp32, BF16x3 and FP16, against the aggregation oracles of test_aggregation_cpu.  No shipped checkpoint was trained
with a sum or a mean: the shipped weights run with the aggregation swapped.

Bounds.  fp32 and BF16x3: max|got - want| <= 1e-3 max(1, max|want|) against float64, the bound of the max's tests in
the relative form a sum needs (a destination's sum grows with its degree).  FP16: the same form against the FP16
oracle, which rounds every tensor-core operand where the kernels do; what remains is fp32 summation order, and an A
element whose fp32 value moves by one ulp rounds to the neighbouring FP16 now and then.  The whole model at FP16 keeps
test_fp16_gpu's 8e-3 (logits) / 4e-3 (boxes): there a last-bit flip of an fp32 sum feeds the next layer's FP16
operand and compounds through a dozen FP16 layers."""
import numpy as np
import pytest
import torch

from test_activations_cpu import NAMES, activate
from test_aggregation_cpu import (_scope_weights, aggregation_oracle, f16_aggregation_oracle, f16_gnn_edge,
                                  f16_pool_edge, segment_reduce)

pytestmark = pytest.mark.gpu
PRECISIONS = ['fp32', 'bf16x3', 'fp16']
CODES = {'fp32': 0, 'bf16x3': 1, 'fp16': 2}


def _lib():
    from pointgnn_b200 import _lib
    return _lib


def _prec(precision):
    if precision != 'fp32' and not _lib().tc_available():
        pytest.skip('tensor-core path needs an sm_90 device')
    return CODES[precision]


def _cuda(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def _err(got, want):
    """max|got - want| over max(1, max|want|)."""
    assert got.shape == want.shape and np.isfinite(got).all()
    return float(np.abs(got - want).max()) / max(1.0, float(np.abs(want).max())) if want.size else 0.0


def _mlp64(h, ws, bs, act='ReLU'):
    for w, b in zip(ws, bs):
        h = activate(act, h @ w.astype(np.float64) + b.astype(np.float64))
    return h


# ---- one edge layer -----------------------------------------------------------------------------------------------
def _layer_case(layer, request):
    """-> (mode, kind, [feat, xyz_src, xyz_dst, dst_index], src, dst, num_dst, ws, bs) with the shipped weights:
    car GNN layer3 on the level-1 graph (features as test_gnn_gpu's _edge_case), car / ped pooling layer1 on the
    level-0 graph."""
    lib = _lib()
    g = request.getfixturevalue('car' if layer in ('gnn', 'car_pool') else 'ped')
    coords, keypoints, edges = g.graph_tuple()
    if layer == 'gnn':
        ws, bs = _scope_weights(g.weights, 'layer3/extract_vertex_features', 2)
        rng = np.random.default_rng(5)
        feat = (np.abs(rng.standard_normal((coords[1].shape[0], ws[0].shape[0] - 3))) * 0.3).astype(np.float32)
        xyz = coords[1].astype(np.float32)
        xyz_dst = (xyz + rng.standard_normal(xyz.shape) * 0.05).astype(np.float32)   # an auto offset
        ed = edges[1]
        return 1, lib.PG_LAYER_EDGE_GNN, [feat, xyz, xyz_dst, None], ed[:, 0], ed[:, 1], len(feat), ws, bs
    lc = g.layer_configs[0]
    ws, bs = _scope_weights(g.weights, 'layer1/extract_vertex_features', len(lc['kwargs']['point_MLP_depth_list']))
    xyz = coords[0].astype(np.float32)
    ed = edges[0]
    return (0, lib.PG_LAYER_EDGE_POOL, [g.graph['intensity'].astype(np.float32), xyz, xyz, keypoints[0][:, 0]],
            ed[:, 0], ed[:, 1], len(keypoints[0]), ws, bs)


def _reference(mode, inputs, src, dst, num_dst, ws, bs, aggregation, precision, act='ReLU'):
    """float64 composition (fp32, BF16x3) or the FP16 oracle (fp16)."""
    feat, xyz_src, xyz_dst, dst_index = inputs
    drow = dst if dst_index is None else dst_index[dst]
    if precision == 'fp16' and mode == 1:
        return f16_gnn_edge(feat, xyz_src, xyz_dst, src, dst, num_dst, ws, bs, act, aggregation)
    if precision == 'fp16':
        return f16_pool_edge(feat, xyz_src, xyz_dst[dst_index], src, dst, num_dst, ws, bs, act, aggregation)
    h = np.concatenate([feat[src], xyz_src[src] - xyz_dst[drow]], axis=1).astype(np.float64)
    return segment_reduce(_mlp64(h, ws, bs, act), dst, num_dst, aggregation)


def _run(mode, kind, inputs, src, dst, num_dst, ws, bs, aggregation, code, act=None, prepared=True, trusted=False):
    lib = _lib()
    feat, xyz_src, xyz_dst, dst_index = inputs
    act = lib.PG_ACT_RELU if act is None else act
    wt, bt = [_cuda(w) for w in ws], [_cuda(b) for b in bs]
    args = (_cuda(feat), _cuda(xyz_src), _cuda(xyz_dst), None if dst_index is None else _cuda(dst_index, torch.int32),
            _cuda(src, torch.int32), _cuda(dst, torch.int32), num_dst)
    if prepared:
        dims = [ws[0].shape[0]] + [w.shape[1] for w in ws]
        layer = lib.PreparedLayer(kind, wt, bt, dims, code, act)
        return layer.edge_mlp_max(*args, trusted=trusted, aggregation=aggregation).cpu().numpy()
    return lib.edge_mlp_max(mode, *args, wt, bt, precision=code, trusted=trusted, activation=act,
                            aggregation=aggregation).cpu().numpy()


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('aggregation', ['sum', 'mean'])
@pytest.mark.parametrize('layer', ['gnn', 'car_pool', 'ped_pool'])
def test_layer(layer, aggregation, precision, request):
    """Prepared and per call; on the tensor cores at bf16x3 and fp16 (counted launches), on the fp32 kernel at fp32."""
    lib = _lib()
    code = _prec(precision)
    mode, kind, inputs, src, dst, num_dst, ws, bs = _layer_case(layer, request)
    want = _reference(mode, inputs, src, dst, num_dst, ws, bs, aggregation, precision)
    tc0 = lib.tc_launch_count(0)
    got = _run(mode, kind, inputs, src, dst, num_dst, ws, bs, aggregation, code)
    assert (lib.tc_launch_count(0) > tc0) == (code != 0)
    err = _err(got, want)
    print('%s %s %s: %.3g (max|want| %.3g)' % (layer, aggregation, precision, err, np.abs(want).max()))
    assert err <= 1e-3, err
    empty = np.bincount(dst, minlength=num_dst) == 0
    assert (got[empty] == 0).all()
    assert _err(_run(mode, kind, inputs, src, dst, num_dst, ws, bs, aggregation, code, prepared=False), want) <= 1e-3


# ---- edge cases, GNN edge layer -----------------------------------------------------------------------------------
def _gnn_edges(rng, nv, hub=7, hub_degree=3000):
    """In-degrees 1 .. 40, vertex 5 without edges, vertex hub with hub_degree edges (dozens of 64-row tiles)."""
    deg = rng.integers(1, 41, nv)
    deg[5] = 0
    deg[hub] = hub_degree
    dst = np.repeat(np.arange(nv), deg)
    return rng.integers(0, nv, dst.size), dst


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('aggregation', ['sum', 'mean'])
def test_gnn_edge_cases(aggregation, precision, request):
    """Empty destinations are exactly 0; a destination with 3000 edges; a foreign edge list in random order, with and
    without the trusted flag; an out-of-range dst raises; E = 0."""
    lib = _lib()
    code = _prec(precision)
    mode, kind, inputs, _, _, nv, ws, bs = _layer_case('gnn', request)
    rng = np.random.default_rng(21)
    src, dst = _gnn_edges(rng, nv)
    want = _reference(mode, inputs, src, dst, nv, ws, bs, aggregation, precision)
    got = _run(mode, kind, inputs, src, dst, nv, ws, bs, aggregation, code)
    assert (got[5] == 0).all()
    assert _err(got, want) <= 1e-3
    perm = rng.permutation(len(src))
    for trusted in (False, True):
        got = _run(mode, kind, inputs, src[perm], dst[perm], nv, ws, bs, aggregation, code, trusted=trusted)
        assert (got[5] == 0).all()
        assert _err(got, want) <= 1e-3, trusted
    bad = dst.copy()
    bad[len(bad) // 2] = nv
    with pytest.raises(lib.PointGNNError, match='out of range'):
        _run(mode, kind, inputs, src, bad, nv, ws, bs, aggregation, code)
    none = np.zeros(0, np.int64)
    got = _run(mode, kind, inputs, none, none, nv, ws, bs, aggregation, code)
    assert got.shape == (nv, ws[-1].shape[1]) and (got == 0).all()


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('name', NAMES)
def test_gnn_sum_every_activation(name, precision, request):
    """Bias and activation per edge, before the sum: biases large enough that act(sum(acc) + b), the max's order,
    fails the bound."""
    from pointgnn_b200.models import gnn
    code = _prec(precision)
    mode, kind, inputs, src, dst, nv, ws, bs = _layer_case('gnn', request)
    bs = [b + 0.5 for b in bs]
    want = _reference(mode, inputs, src, dst, nv, ws, bs, 'sum', precision, act=name)
    got = _run(mode, kind, inputs, src, dst, nv, ws, bs, 'sum', code, act=gnn.activation_fn_dict[name])
    err = _err(got, want)
    assert err <= 1e-3, (name, err)
    feat, xyz_src, xyz_dst, _ = inputs
    h = _mlp64(np.concatenate([feat[src], xyz_src[src] - xyz_dst[dst]], axis=1), ws[:1], bs[:1], name)
    acc = segment_reduce(h @ ws[1].astype(np.float64), dst, nv, 'sum')
    wrong = activate(name, acc + bs[1].astype(np.float64))
    wrong[np.bincount(dst, minlength=nv) == 0] = 0
    assert _err(wrong, want) > 10 * 1e-3, name


# ---- fused against op by op, and the prepared handle ----------------------------------------------------------------
def _user_sum(point_features, point_centers, num_centers):
    """A user-written aggregation: the same sum, but not the package's function, so the layer runs op by op."""
    from pointgnn_b200.models import gnn
    return gnn.graph_scatter_sum_fn(point_features, point_centers, num_centers)


def _apply(g, scope, aggregation_fn, precision, store=None):
    import pointgnn_b200
    from pointgnn_b200.models import gnn
    coords, keypoints, edges = g.graph_tuple()
    lc = [c for c in g.layer_configs if c['scope'] == scope][0]
    store = store or gnn.VariableStore(g.weights)
    pointgnn_b200.set_precision(precision)
    try:
        with gnn.variable_session(store), gnn.variable_scope(scope):
            if scope == 'layer1':
                return gnn.PointSetPooling(aggregation_fn=aggregation_fn).apply_regular(
                    _cuda(g.graph['intensity']), _cuda(coords[0]), _cuda(keypoints[0], torch.int32),
                    _cuda(edges[0], torch.int32), **lc['kwargs']).cpu().numpy()
            rng = np.random.default_rng(5)
            feat = (np.abs(rng.standard_normal((coords[1].shape[0], 300))) * 0.3).astype(np.float32)
            return gnn.GraphNetAutoCenter(aggregation_fn=aggregation_fn).apply_regular(
                _cuda(feat), _cuda(coords[1].astype(np.float32)), None, _cuda(edges[1], torch.int32),
                **lc['kwargs']).cpu().numpy()
    finally:
        pointgnn_b200.set_precision('fp32')


@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
@pytest.mark.parametrize('scope', ['layer1', 'layer3'])
def test_fused_vs_op_by_op(scope, precision, car):
    from pointgnn_b200.models import gnn
    _prec(precision)
    lib = _lib()
    tc0 = lib.tc_launch_count(0)
    fused = _apply(car, scope, gnn.graph_scatter_sum_fn, precision)
    tc1 = lib.tc_launch_count(0)
    by_op = _apply(car, scope, _user_sum, precision)
    assert lib.tc_launch_count(0) == tc1 and (tc1 > tc0) == (precision != 'fp32')
    assert _err(fused, by_op) <= 1e-3


def test_one_prepared_handle_serves_every_aggregation(car):
    """store.prepared does not grow when only the aggregation changes, and each call still reduces its own way."""
    from pointgnn_b200.models import gnn
    _prec('bf16x3')
    store = gnn.VariableStore(car.weights)
    for scope in ('layer1', 'layer3'):
        first = _apply(car, scope, gnn.graph_scatter_max_fn, 'bf16x3', store)
        n = len(store.prepared)
        outs = [_apply(car, scope, fn, 'bf16x3', store) for fn in
                (gnn.graph_scatter_sum_fn, gnn.graph_scatter_mean_fn, gnn.graph_scatter_max_fn)]
        assert len(store.prepared) == n, scope
        assert np.array_equal(outs[2], first)     # the max reads no sum state: bit for bit
        assert _err(outs[0], first) > 1e-2 and _err(outs[1], outs[0]) > 1e-2, scope


# ---- the whole model --------------------------------------------------------------------------------------------
def _predict(g, aggregation_fn, precision):
    import pointgnn_b200
    from pointgnn_b200.models import gnn, models
    coords, keypoints, edges = g.graph_tuple()
    pointgnn_b200.set_precision(precision)
    try:
        model = models.get_model(g.config['model_name'])(num_classes=g.config['num_classes'], box_encoding_len=7,
                                                         mode='test', **g.config['model_kwargs'])
        model._default_layers_type['scatter_max_point_set_pooling'] = gnn.PointSetPooling(aggregation_fn=aggregation_fn)
        model._default_layers_type['scatter_max_graph_auto_center_net'] = gnn.GraphNetAutoCenter(
            aggregation_fn=aggregation_fn)
        model.load_weights(g.weights)
        logits, boxes = model.predict(g.graph['intensity'], coords, keypoints, edges, is_training=True)
    finally:
        pointgnn_b200.set_precision('fp32')
    return np.asarray(logits), np.asarray(boxes)


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('aggregation', ['sum', 'mean'])
@pytest.mark.parametrize('model', ['car', 'ped'])
def test_whole_model(model, aggregation, precision, request):
    """Both layer types with graph_scatter_{sum,mean}_fn.  The sum is not run at FP16: sums grow through the three
    iterations past FP16's 65504, where the operands saturate."""
    from pointgnn_b200.models import gnn
    if aggregation == 'sum' and precision == 'fp16':
        pytest.skip('sums exceed the FP16 range')
    _prec(precision)
    g = request.getfixturevalue(model)
    coords, keypoints, edges = g.graph_tuple()
    args = (g.weights, g.layer_configs, g.config['num_classes'], 7, g.graph['intensity'], coords, keypoints, edges)
    if precision == 'fp16':
        with f16_aggregation_oracle(aggregation) as o:
            want_l, want_b = o.predict(*args)
    else:
        with aggregation_oracle(aggregation) as o:
            want_l, want_b = o.predict(*args)
    logits, boxes = _predict(g, getattr(gnn, 'graph_scatter_%s_fn' % aggregation), precision)
    if precision == 'fp16':
        el, eb = np.abs(logits - want_l).max(), np.abs(boxes - want_b).max()
        assert el <= 8e-3 and eb <= 4e-3, (el, eb)
    else:
        el, eb = _err(logits, want_l), _err(boxes, want_b)
        assert el <= 1e-3 and eb <= 1e-3, (el, eb)
    print('%s %s %s: logits %.3g boxes %.3g (max|logits| %.3g)' % (model, aggregation, precision, el, eb,
                                                                    np.abs(want_l).max()))

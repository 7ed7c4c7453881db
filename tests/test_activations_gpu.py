"""Every activation of the reference's table through the dense, pooling, GNN edge and predictor layers and the whole
model, at both precisions, against the oracle (oracle/gnn.py) with each activation."""
import ctypes
from functools import partial

import numpy as np
import pytest
import torch

from oracle import gnn as ognn
from oracle.gnn import NAMES, activate
from test_activations_cpu import with_activation

pytestmark = pytest.mark.gpu
FLT_MIN = np.finfo(np.float32).min
PRECISIONS = ['fp32', 'bf16x3']


def _lib():
    from pointgnn_b200 import _lib
    return _lib


def _code(name):
    from pointgnn_b200.models import gnn
    return gnn.activation_fn_dict[name]


def _prec(precision):
    if precision == 'bf16x3' and not _lib().tc_available():
        pytest.skip('tensor-core path needs an sm_90 device')
    return 0 if precision == 'fp32' else 1


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _close(got, want, what, scale_with_output=False):
    empty = want == FLT_MIN
    assert np.array_equal(got == FLT_MIN, empty), what
    if (~empty).any():
        scale = max(1.0, float(np.abs(want[~empty]).max())) if scale_with_output else 1.0
        err = float(np.abs(got - want)[~empty].max())
        assert err < 1e-3 * scale, (what, err, scale)
        return err
    return 0.0


def _layers(rng, dims, bias=0.1):
    ws = [(rng.standard_normal((dims[i], dims[i + 1])) / np.sqrt(dims[i])).astype(np.float32) for i in range(len(dims) - 1)]
    bs = [(rng.standard_normal(dims[i + 1]) * bias).astype(np.float32) for i in range(len(dims) - 1)]
    return ws, bs


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('name', NAMES)
def test_dense_mlp(name, precision):
    """FFMA-only (K < 64), one tensor-core block (N = 300), column blocks (N = 512); is_logits and residual."""
    lib = _lib()
    p = _prec(precision)
    rng = np.random.default_rng(7)
    for k, n in ((32, 4), (300, 300), (64, 512)):
        dims = [k, 128, n]
        ws, bs = _layers(rng, dims)
        x = (rng.standard_normal((1000, k)) * 2).astype(np.float32)
        res = rng.standard_normal((1000, n)).astype(np.float32)
        layer = lib.PreparedLayer(lib.PG_LAYER_MLP, [_cuda(w) for w in ws], [_cuda(b) for b in bs], dims, p, _code(name))
        for logits in (False, True):
            for residual in (None, res):
                h = activate(name, x @ ws[0] + bs[0])
                want = h @ ws[1] + bs[1]
                want = want if logits else activate(name, want)
                if residual is not None:
                    want = want + residual
                got = layer.mlp(_cuda(x), last_linear=logits,
                                residual=None if residual is None else _cuda(residual)).cpu().numpy()
                _close(got, want, (name, k, n, logits, residual is not None))
    # the per-call entry point takes the code too
    got = lib.fully_connected(_cuda(x), _cuda(ws[0]), _cuda(bs[0]), True, precision=p, activation=_code(name))
    _close(got.cpu().numpy(), activate(name, x @ ws[0] + bs[0]), name)


def _pool_case(rng, dims, e, nv=900, nk=400):
    ws, bs = _layers(rng, dims)
    dst = np.sort(np.concatenate([rng.integers(0, nk, e // 2), rng.integers(10, 14, e - e // 2)]))
    src = rng.integers(0, nv, e)
    f = rng.random((nv, 1)).astype(np.float32)
    x = (rng.standard_normal((nv, 3)) * 5).astype(np.float32)
    kp = rng.integers(0, nv, nk)
    h0 = np.concatenate([f[src], x[src] - x[kp[dst]]], axis=1)
    args = (_cuda(f), _cuda(x), _cuda(x), _cuda(kp.astype(np.int32)), _cuda(src.astype(np.int32)),
            _cuda(dst.astype(np.int32)), nk, [_cuda(w) for w in ws], [_cuda(b) for b in bs])
    return args, h0, ws, bs, dst, nk


def _mlp_max(name, h, ws, bs, dst, nk):
    for w, b in zip(ws, bs):
        h = activate(name, h @ w + b)
    return ognn.graph_scatter_max_fn(h, dst, nk)


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('name', NAMES)
def test_pooling_edge_layer(name, precision):
    """The car chain, the ped chain (wide last layer) and an odd-width chain with pad columns."""
    lib = _lib()
    p = _prec(precision)
    rng = np.random.default_rng(11)
    for dims in ((4, 32, 64, 128, 300), (4, 32, 64, 128, 256, 512), (4, 20, 36, 300)):
        args, h0, ws, bs, dst, nk = _pool_case(rng, dims, 5000)
        got = lib.edge_mlp_max(0, *args, precision=p, activation=_code(name)).cpu().numpy()
        _close(got, _mlp_max(name, h0, ws, bs, dst, nk), (name, dims))


def _gnn_case(rng, c=300, n=300, nv=3000, neg_bias=False):
    """In-degrees 1 .. 40 (uniform-warp and segmented flushes), vertex 5 without edges."""
    deg = rng.integers(1, 41, nv)
    deg[5] = 0
    dst = np.repeat(np.arange(nv), deg)
    src = rng.integers(0, nv, dst.size)
    feat = rng.standard_normal((nv, c)).astype(np.float32)
    xyz = (rng.standard_normal((nv, 3)) * 3).astype(np.float32)
    ws, bs = _layers(rng, (c + 3, n, n))
    if neg_bias:
        bs[1] = bs[1] - 20.0      # whole destinations with only negative outputs
    h0 = np.concatenate([feat[src], xyz[src] - xyz[dst]], axis=1)
    args = (_cuda(feat), _cuda(xyz), _cuda(xyz), None, _cuda(src.astype(np.int32)), _cuda(dst.astype(np.int32)), nv,
            [_cuda(w) for w in ws], [_cuda(b) for b in bs])
    return args, h0, ws, bs, dst, nv


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('name', NAMES)
def test_gnn_edge_layer(name, precision):
    lib = _lib()
    p = _prec(precision)
    rng = np.random.default_rng(13)
    for neg in (False, True):
        args, h0, ws, bs, dst, nv = _gnn_case(rng, neg_bias=neg)
        want = _mlp_max(name, h0, ws, bs, dst, nv)
        got = lib.edge_mlp_max(1, *args, precision=p, activation=_code(name)).cpu().numpy()
        assert (got[5] == FLT_MIN).all()
        if neg and name in ('NONE', 'Tanh', 'LeakyReLU', 'ELU'):
            assert (want[want != FLT_MIN] < 0).mean() > 0.5
        _close(got, want, (name, neg))
        if p == 1:    # the max is exact and the flush order does not matter: two runs agree bit for bit
            again = lib.edge_mlp_max(1, *args, precision=p, activation=_code(name)).cpu().numpy()
            assert np.array_equal(got, again)


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('name', NAMES)
def test_predictor_fast_path(name, precision):
    import pointgnn_b200
    from pointgnn_b200.models import gnn
    _prec(precision)
    rng = np.random.default_rng(17)
    d, c, box = 300, 4, 7
    for h in (64, 128):
        weights = {}
        for scope, shapes in [('predictor/cls', [(d, h), (h, c)])] + [
                ('predictor/loc/cls_%d' % i, [(d, h), (h, h), (h, box)]) for i in range(c)]:
            for j, (a, b) in enumerate(shapes):
                base = scope + '/' + ('fully_connected' if j == 0 else 'fully_connected_%d' % j)
                weights[base + '/weights'] = (rng.standard_normal((a, b)) / np.sqrt(a)).astype(np.float32)
                weights[base + '/biases'] = (rng.standard_normal(b) * 0.1).astype(np.float32)
        x = rng.standard_normal((700, d)).astype(np.float32)
        want_l, want_b = ognn.class_aware_predictor(weights, '', x, c, box, activation_type=name, cls_Ks=(h,),
                                                    loc_Ks=(h, h))
        pointgnn_b200.set_precision(precision)
        try:
            pred = gnn.ClassAwarePredictor(partial(gnn.multi_layer_fc_fn, Ks=(h,), num_layer=2),
                                           partial(gnn.multi_layer_fc_fn, Ks=(h, h), num_layer=3))
            with gnn.variable_session(gnn.VariableStore(weights)):
                logits, boxes = pred.apply_regular(_cuda(x), c, box, normalization_type='NONE', activation_type=name)
        finally:
            pointgnn_b200.set_precision('fp32')
        _close(logits.cpu().numpy(), want_l, (name, h))
        _close(boxes.cpu().numpy(), want_b, (name, h))


def _model(g, layer_configs, precision):
    import pointgnn_b200
    from pointgnn_b200.models import models
    coords, keypoints, edges = g.graph_tuple()
    pointgnn_b200.set_precision(precision)
    try:
        model = models.get_model(g.config['model_name'])(
            num_classes=g.config['num_classes'], box_encoding_len=7, mode='test',
            **dict(g.config['model_kwargs'], layer_configs=layer_configs))
        model.load_weights(g.weights)
        return model.predict(g.graph['intensity'], coords, keypoints, edges, is_training=True)
    finally:
        pointgnn_b200.set_precision('fp32')


MIXED = {'edge_MLP_activation_type': 'ELU', 'update_MLP_activation_type': 'Tanh',
         'auto_offset_MLP_feature_activation_type': 'LeakyReLU', 'point_MLP_activation_type': 'Sigmoid',
         'output_MLP_activation_type': 'ReLU', 'activation_type': 'ReLU6'}


@pytest.mark.parametrize('precision', PRECISIONS)
@pytest.mark.parametrize('name', NAMES + ['mixed'])
@pytest.mark.parametrize('model', ['car', 'ped'])
def test_whole_model(model, name, precision, request):
    """Every *_activation_type of the config set to one activation, or each MLP to its own (mixed)."""
    _prec(precision)
    g = request.getfixturevalue(model)
    lcs = with_activation(g.layer_configs, per_key=MIXED) if name == 'mixed' else with_activation(g.layer_configs, name)
    coords, keypoints, edges = g.graph_tuple()
    want_l, want_b = ognn.predict(g.weights, lcs, g.config['num_classes'], 7, g.graph['intensity'], coords, keypoints,
                                  edges)
    logits, boxes = _model(g, lcs, precision)
    err = max(_close(logits, want_l, name, True), _close(boxes, want_b, name, True))
    print('max |err| %s %s %s: %.3g' % (model, name, precision, err))


def test_prepared_cache_key_includes_the_activation(car):
    """One VariableStore, the same variables with ReLU then ELU: each result matches its own oracle."""
    import pointgnn_b200
    from pointgnn_b200.models import gnn
    _prec('bf16x3')
    rng = np.random.default_rng(3)
    weights = {'l/fully_connected/weights': rng.standard_normal((64, 300)).astype(np.float32) / 8,
               'l/fully_connected/biases': rng.standard_normal(300).astype(np.float32)}
    x = rng.standard_normal((500, 64)).astype(np.float32)
    store = gnn.VariableStore(weights)
    pointgnn_b200.set_precision('bf16x3')
    try:
        for name in ('ReLU', 'ELU', 'ReLU'):
            with gnn.variable_session(store), gnn.variable_scope('l'):
                got = gnn.multi_layer_neural_network_fn(_cuda(x), Ks=(300,), normalization_type='NONE',
                                                        activation_type=name)
            want = activate(name, x @ weights['l/fully_connected/weights'] + weights['l/fully_connected/biases'])
            _close(got.cpu().numpy(), want, name)
    finally:
        pointgnn_b200.set_precision('fp32')
    assert len(store.prepared) == 2


def test_out_of_range_activation_codes_are_errors():
    lib = _lib()
    w, b = _cuda(np.ones((8, 8), np.float32)), _cuda(np.zeros(8, np.float32))
    for code in (7, 255, 256, 1 << 40, -1):
        with pytest.raises(lib.PointGNNError):
            lib.PreparedLayer(lib.PG_LAYER_MLP, [w], [b], [8, 8], 0, code)
        with pytest.raises(lib.PointGNNError):
            lib.fully_connected(_cuda(np.ones((4, 8), np.float32)), w, b, True, activation=code)
    # the ABI itself rejects a code whose bits lie above the 8-bit field
    for word in (lib.PG_FLAG_ACTIVATION | (256 << lib.PG_ACT_SHIFT), lib.PG_FLAG_ACTIVATION | (7 << lib.PG_ACT_SHIFT)):
        handle = ctypes.c_void_p()
        wp = (ctypes.c_void_p * 1)(w.data_ptr())
        bp = (ctypes.c_void_p * 1)(b.data_ptr())
        dm = (lib.c_i32 * 2)(8, 8)
        assert lib.load().pg_layer_create(lib.PG_LAYER_MLP, wp, bp, dm, 1, word, None, ctypes.byref(handle)) == -1

"""The FP16 precision (code 2, ``set_precision('fp16')``) on the GPU against the FP16 oracle (oracle/gnn.py with
``fp16=True``): the dense kernel, the pooling and GNN edge layers (prepared and per call, car and ped), every non-ReLU
activation of the GNN edge layer, the whole model on all seven checkpoints, saturation at FP16's range, and the
rejected precision codes.

Bounds.  Dense layers: 1e-4, both sides round the same operands and only the fp32 summation order differs.  Edge
layers: 1e-3 of the output's scale (max(1, max |want|)), since an fp32 pre-rounding value that differs in its last
bit may round to the neighbouring FP16.  Whole model: 2e-2 on logits / 1e-2 on boxes of the fp32 golden, the accuracy
FP16 gives up, and 8e-3 / 4e-3 of the FP16 oracle.  The latter is what the arithmetic allows, not a slack: such flips
compound through a dozen FP16 layers, and the oracle itself moves by 1.6e-3 (car_auto_T0) to 2.9e-3 (car_auto_T3) on
logits when only pooling layer 0's fp32 sums are rounded differently (float64 then fp32, instead of fp32); the kernels
measured 2.2e-3 to 4.2e-3 on logits and <= 1.6e-3 on boxes on an H100."""
import numpy as np
import pytest
import torch

from conftest import ALL_CHECKPOINTS, load_golden
from oracle import gnn as ognn

pytestmark = pytest.mark.gpu
FLT_MIN = np.finfo(np.float32).min
FP16 = 2


def _lib():
    from pointgnn_b200 import _lib
    if not _lib.tc_available():
        pytest.skip('tensor-core path needs an sm_90 device')
    return _lib


def _cuda(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def _close(got, want, what, tol=1e-3):
    empty = want == FLT_MIN
    assert np.array_equal(got == FLT_MIN, empty), what
    assert np.isfinite(got).all(), what
    scale = max(1.0, float(np.abs(want[~empty]).max())) if (~empty).any() else 1.0
    err = float(np.abs(got - want)[~empty].max()) if (~empty).any() else 0.0
    assert err <= tol * scale, (what, err, scale)
    return err


def test_fully_connected_vs_oracle():
    lib = _lib()
    rng = np.random.default_rng(1)
    dense0 = lib.tc_launch_count(1)
    for m, k, n in ((1, 1, 1), (257, 300, 300), (1000, 303, 300), (77, 64, 3), (513, 4, 32), (130, 512, 256),
                    (64, 300, 7), (255, 256, 256), (256, 300, 64), (4099, 300, 320), (33, 128, 300), (700, 512, 300)):
        x = rng.standard_normal((m, k)).astype(np.float32)
        w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
        b = rng.standard_normal(n).astype(np.float32)
        r = rng.standard_normal((m, n)).astype(np.float32)
        for relu in (True, False):
            for res in (None, r):
                want = ognn.dense(x, w, b, 'ReLU' if relu else 'NONE', fp16=True)
                want = want if res is None else want + res
                got = lib.fully_connected(_cuda(x), _cuda(w), _cuda(b), relu, residual=None if res is None else _cuda(res),
                                          precision=FP16).cpu().numpy()
                assert got.shape == want.shape and np.abs(got - want).max() <= 1e-4, (m, k, n, relu)
    # the wide shapes ran on the FP16 tensor-core kernel (as in test_gnn_gpu's BF16x3 count)
    assert lib.tc_launch_count(1) - dense0 >= 4 * 4 + 2 * 4 * 2


def _mlp_weights(g, scope, n):
    names = ['fully_connected'] + ['fully_connected_%d' % i for i in range(1, n)]
    ws = [g.weights['%s/%s/weights' % (scope, s)] for s in names]
    bs = [g.weights['%s/%s/biases' % (scope, s)] for s in names]
    return ws, bs


def _run_edge(lib, kind, mode, ws, bs, feats, xyz_src, xyz_dst, dst_index, src, dst, num_dst, prepared, act=None):
    dims = [ws[0].shape[0]] + [w.shape[1] for w in ws]
    cw, cb = [_cuda(w) for w in ws], [_cuda(b) for b in bs]
    args = (_cuda(feats), _cuda(xyz_src), _cuda(xyz_dst), None if dst_index is None else _cuda(dst_index, torch.int32),
            _cuda(src, torch.int32), _cuda(dst, torch.int32), num_dst)
    a = lib.PG_ACT_RELU if act is None else act
    if prepared:
        layer = lib.PreparedLayer(kind, cw, cb, dims, FP16, a)
        return layer.edge_mlp_max(*args).cpu().numpy()
    return lib.edge_mlp_max(mode, *args, cw, cb, precision=FP16, activation=a).cpu().numpy()


@pytest.mark.parametrize('prepared', [True, False])
@pytest.mark.parametrize('name', ['car_auto_T3_train', 'ped_cyl_auto_T3_trainval'])
def test_pooling_edge_layer(name, prepared):
    lib = _lib()
    g = load_golden(name)
    coords, keypoints, edges = g.graph_tuple()
    lc = g.layer_configs[0]
    ws, bs = _mlp_weights(g, 'layer1/extract_vertex_features', len(lc['kwargs']['point_MLP_depth_list']))
    kp = keypoints[0][:, 0]
    ed = edges[0]
    feats = g.graph['intensity'].astype(np.float32)
    want = ognn.pool_edge_layer(feats, coords[0], coords[0][kp], ed[:, 0], ed[:, 1], len(kp), ws, bs, fp16=True)
    seg0 = lib.tc_launch_count(0)
    got = _run_edge(lib, lib.PG_LAYER_EDGE_POOL, lib.PG_EDGE_POOL, ws, bs, feats, coords[0], coords[0], kp,
                    ed[:, 0], ed[:, 1], len(kp), prepared)
    assert lib.tc_launch_count(0) > seg0
    print('%s pooling (prepared %s): max |err| %.3g' % (name, prepared, _close(got, want, name)))


@pytest.mark.parametrize('prepared', [True, False])
@pytest.mark.parametrize('name', ['car_auto_T3_train', 'ped_cyl_auto_T3_trainval'])
def test_gnn_edge_layer(name, prepared):
    lib = _lib()
    g = load_golden(name)
    coords, _, edges = g.graph_tuple()
    lc = [l for l in g.layer_configs if l['scope'] == 'layer2'][0]
    ws, bs = _mlp_weights(g, 'layer2/extract_vertex_features', len(lc['kwargs']['edge_MLP_depth_list']))
    k = coords[1].shape[0]
    rng = np.random.default_rng(5)
    feats = np.abs(rng.standard_normal((k, ws[0].shape[0] - 3))).astype(np.float32) * 0.3
    xyz = coords[1].astype(np.float32)
    xyz_dst = xyz + (rng.standard_normal(xyz.shape) * 0.05).astype(np.float32)    # an auto offset
    ed = edges[1]
    want = ognn.gnn_edge_layer(feats, xyz, xyz_dst, ed[:, 0], ed[:, 1], k, ws, bs, fp16=True)
    seg0 = lib.tc_launch_count(0)
    got = _run_edge(lib, lib.PG_LAYER_EDGE_GNN, lib.PG_EDGE_GNN, ws, bs, feats, xyz, xyz_dst, None, ed[:, 0], ed[:, 1],
                    k, prepared)
    assert lib.tc_launch_count(0) > seg0
    print('%s GNN edge layer (prepared %s): max |err| %.3g' % (name, prepared, _close(got, want, name)))


@pytest.mark.parametrize('name', ['NONE', 'ReLU6', 'LeakyReLU', 'ELU', 'Sigmoid', 'Tanh'])
def test_gnn_edge_layer_activations(name):
    """wg_gemm_act_f16_kernel: the GNN edge layer with every other activation of the reference's table, including
    destinations whose outputs are all negative (the sign-aware segment max)."""
    from pointgnn_b200.models import gnn
    lib = _lib()
    rng = np.random.default_rng(13)
    nv, c, n = 700, 64, 128
    dst = np.sort(rng.integers(0, nv, 9000))
    dst = dst[dst != 5]                     # an empty destination
    src = rng.integers(0, nv, dst.size)
    feat = rng.standard_normal((nv, c)).astype(np.float32)
    xyz = (rng.standard_normal((nv, 3)) * 3).astype(np.float32)
    ws = [(rng.standard_normal((c + 3, n)) / np.sqrt(c + 3)).astype(np.float32),
          (rng.standard_normal((n, n)) / np.sqrt(n)).astype(np.float32)]
    for neg in (False, True):
        bs = [(rng.standard_normal(n) * 0.1).astype(np.float32), (rng.standard_normal(n) * 0.1).astype(np.float32)]
        if neg:
            bs[1] = bs[1] - 20.0
        want = ognn.gnn_edge_layer(feat, xyz, xyz, src, dst, nv, ws, bs, act=name, fp16=True)
        act = gnn.activation_fn_dict[name]
        for prepared in (False, True):
            got = _run_edge(lib, lib.PG_LAYER_EDGE_GNN, lib.PG_EDGE_GNN, ws, bs, feat, xyz, xyz, None, src, dst, nv,
                            prepared, act=act)
            assert (got[5] == FLT_MIN).all()
            _close(got, want, (name, neg, prepared))


def _predict(g, precision, model=None):
    import pointgnn_b200
    from pointgnn_b200.models import models
    coords, keypoints, edges = g.graph_tuple()
    pointgnn_b200.set_precision(precision)
    try:
        if model is None:
            model = models.get_model(g.config['model_name'])(num_classes=g.config['num_classes'], box_encoding_len=7,
                                                             mode='test', **g.config['model_kwargs'])
            model.load_weights(g.weights)
        logits, boxes = model.predict(g.graph['intensity'], coords, keypoints, edges, is_training=True)
    finally:
        pointgnn_b200.set_precision('fp32')
    return np.asarray(logits), np.asarray(boxes), model


@pytest.mark.parametrize('name', ALL_CHECKPOINTS)
def test_predict_every_checkpoint(name):
    lib = _lib()
    g = load_golden(name)
    coords, keypoints, edges = g.graph_tuple()
    want_l, want_b = ognn.predict(g.weights, g.layer_configs, g.config['num_classes'], 7, g.graph['intensity'], coords,
                                  keypoints, edges, fp16=True)
    tc0 = (lib.tc_launch_count(0), lib.tc_launch_count(1))
    logits, boxes, _ = _predict(g, 'fp16')
    assert lib.tc_launch_count(0) > tc0[0] and lib.tc_launch_count(1) > tc0[1]
    el, eb = np.abs(logits - want_l).max(), np.abs(boxes - want_b).max()
    gl, gb = np.abs(logits - g.gnn['logits']).max(), np.abs(boxes - g.gnn['boxes']).max()
    print('%s: vs FP16 oracle %.3g / %.3g, vs fp32 golden %.3g / %.3g' % (name, el, eb, gl, gb))
    assert el <= 8e-3 and eb <= 4e-3, (name, el, eb)
    assert gl <= 2e-2 and gb <= 1e-2, (name, gl, gb)


def test_precisions_never_share_a_prepared_layer():
    """One model, switched between bf16x3 and fp16: each arithmetic gets its own prepared layers and its own answer."""
    _lib()
    g = load_golden('car_auto_T3_train')
    l_bf, b_bf, model = _predict(g, 'bf16x3')
    l_16, b_16, _ = _predict(g, 'fp16', model)
    l_bf2, _, _ = _predict(g, 'bf16x3', model)
    keys = model._store.prepared.keys()
    assert {k[3] for k in keys} == {1, 2}
    assert len([k for k in keys if k[3] == 1]) == len([k for k in keys if k[3] == 2])
    assert np.array_equal(l_bf, l_bf2)
    assert np.abs(l_bf - g.gnn['logits']).max() < 1e-3
    assert np.abs(l_16 - l_bf).max() > 1e-4          # the FP16 layers really ran


def test_saturation():
    """Operands beyond FP16's range clamp to +-65504 instead of becoming inf."""
    lib = _lib()
    rng = np.random.default_rng(3)
    m, k, n = 300, 128, 64
    x = rng.standard_normal((m, k)).astype(np.float32)
    x[::7, ::5] = 1e5
    x[3::11, 1::9] = -3e6
    w = (rng.standard_normal((k, n)) * 1e-3).astype(np.float32)
    w[5, :] = 7e4
    w[9, ::3] = -1e9
    b = rng.standard_normal(n).astype(np.float32)
    want = ognn.dense(x, w, b, 'NONE', fp16=True)
    got = lib.fully_connected(_cuda(x), _cuda(w), _cuda(b), False, precision=FP16).cpu().numpy()
    assert np.isfinite(got).all() and np.isfinite(want).all()
    assert np.abs(want).max() > 1e9                  # the clamped values really are in play
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5 * np.abs(want).max())
    # the same through the GNN edge kernel's register-built A: features beyond the range
    # (hoisted P GEMM: feature 7 clamps; P beyond the range: the edge kernel's A clamps)
    feat = rng.standard_normal((50, 60)).astype(np.float32)
    feat[::3, 7] = 2e5
    xyz = rng.standard_normal((50, 3)).astype(np.float32)
    dst = np.sort(rng.integers(0, 50, 900))
    src = rng.integers(0, 50, 900)
    ws = [(rng.standard_normal((63, 64)) * 0.05).astype(np.float32), (rng.standard_normal((64, 64)) * 0.05).astype(np.float32)]
    ws[0][7, :] = 3.0
    bs = [np.zeros(64, np.float32), np.zeros(64, np.float32)]
    want = ognn.gnn_edge_layer(feat, xyz, xyz, src, dst, 50, ws, bs, fp16=True)
    got = _run_edge(lib, lib.PG_LAYER_EDGE_GNN, lib.PG_EDGE_GNN, ws, bs, feat, xyz, xyz, None, src, dst, 50, False)
    _close(got, want, 'edge saturation')


def test_precision_code_3_rejected():
    lib = _lib()
    x = torch.ones((4, 64), device='cuda')
    w = torch.ones((64, 64), device='cuda')
    b = torch.zeros(64, device='cuda')
    for call in (lambda: lib.fully_connected(x, w, b, True, precision=3),
                 lambda: lib.PreparedLayer(lib.PG_LAYER_MLP, [w], [b], [64, 64], 3),
                 lambda: lib.edge_mlp_max(lib.PG_EDGE_GNN, torch.ones((4, 61), device='cuda'), x[:, :3].contiguous(),
                                          x[:, :3].contiguous(), None, torch.zeros(4, dtype=torch.int32, device='cuda'),
                                          torch.zeros(4, dtype=torch.int32, device='cuda'), 4, [w, w], [b, b],
                                          precision=3)):
        with pytest.raises(lib.PointGNNError) as e:
            call()
        assert e.value.code == lib.PG_ERR_INVALID_ARGUMENT
        # the exception carries pg_last_error()'s text
        assert 'unknown precision 3' in str(e.value)
        assert 'unknown precision 3' in lib.load().pg_last_error().decode()

"""GPU parity tests for the GNN half: CUDA kernels (through the C ABI / the reference-shaped
Python layer API) vs the fp32 CPU oracle, with the reference's trained weights.

Tolerance (BASELINE.json north_star): vertex features / logits / box encodings within 1e-3
absolute of the fp32 CPU path.  The fp32 FFMA kernels are expected ~1e-5; the wgmma BF16x3
kernels ~1e-4 (three-term split, see DESIGN.md)."""
import numpy as np
import pytest
import torch

from conftest import ALL_CHECKPOINTS, load_golden
from oracle import gnn as ognn
from oracle import graph as ograph
from oracle import synth

pytestmark = pytest.mark.gpu
TOL = 1e-3
PRECISIONS = ['fp32', 'bf16x3']


def _need(precision):
    from pointgnn_b200 import _lib
    if precision == 'bf16x3' and not _lib.tc_available():
        pytest.skip('tensor-core path needs an sm_90 device')


def _cuda(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def test_scatter_max_vs_oracle():
    from pointgnn_b200.models import gnn
    rng = np.random.default_rng(0)
    for e, c, k, sorted_ids in ((1000, 300, 37, True), (5000, 7, 600, False), (64, 1, 3, True), (3, 513, 5, False)):
        f = rng.standard_normal((e, c)).astype(np.float32)
        ids = rng.integers(0, k, e)
        if sorted_ids:
            ids = np.sort(ids)
        out = gnn.graph_scatter_max_fn(_cuda(f), _cuda(ids.astype(np.int32)), k).cpu().numpy()
        assert np.array_equal(out, ognn.graph_scatter_max_fn(f, ids, k))      # max is exact
    # empty input, every segment empty -> float lowest
    out = gnn.graph_scatter_max_fn(torch.zeros((0, 4), device='cuda'), torch.zeros(0, dtype=torch.int32, device='cuda'), 3)
    assert np.array_equal(out.cpu().numpy(), np.full((3, 4), np.finfo(np.float32).min, np.float32))
    # int64 [E,1] ids as the reference passes them
    f = rng.standard_normal((10, 2)).astype(np.float32)
    ids = np.array([0, 0, 1, 1, 1, 4, 4, 4, 4, 4])
    out = gnn.graph_scatter_max_fn(_cuda(f), _cuda(ids[:, None]), 5).cpu().numpy()
    assert np.array_equal(out, ognn.graph_scatter_max_fn(f, ids, 5))


@pytest.mark.parametrize('precision', PRECISIONS)
def test_fully_connected_vs_oracle(precision):
    """pg_fully_connected alone (NumPy fp32 as the checker): odd shapes, row tails (m % 256 != 0), K not a
    multiple of 16, N < 8 heads, bias / ReLU / residual combinations - for the FFMA kernel and for the
    wgmma BF16x3 dense kernel (which must really run for the wide shapes)."""
    _need(precision)
    import pointgnn_b200
    from pointgnn_b200 import _lib
    pointgnn_b200.set_precision(precision)
    rng = np.random.default_rng(1)
    tol = 1e-4 if precision == 'fp32' else 3e-4
    dense0 = _lib.tc_launch_count(1)
    for m, k, n in ((1, 1, 1), (257, 300, 300), (1000, 303, 300), (77, 64, 3), (513, 4, 32), (130, 512, 256),
                    (64, 300, 7), (255, 256, 256), (256, 300, 64), (4099, 300, 320), (33, 128, 300), (700, 512, 300)):
        x = rng.standard_normal((m, k)).astype(np.float32)
        w = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
        b = rng.standard_normal(n).astype(np.float32)
        r = rng.standard_normal((m, n)).astype(np.float32)
        for relu in (True, False):
            for res in (None, r):
                want = x @ w + b
                if relu:
                    want = np.maximum(want, 0)
                if res is not None:
                    want = want + res
                got = _lib.fully_connected(_cuda(x), _cuda(w), _cuda(b), relu, residual=None if res is None else _cuda(res),
                                           precision=pointgnn_b200.get_precision()).cpu().numpy()
                assert got.shape == want.shape and np.abs(got - want).max() < tol, (m, k, n, relu)
    if precision == 'bf16x3':
        # (257,300,300), (255,256,256), (256,300,64), (33,128,300) x 4 bias/residual combinations; the others are
        # K % 4 != 0, K < 64 or N < 8 and take the FFMA kernel; (130,512,256), (700,512,300) add one launch per
        # call and (4099,300,320) is wider than one launch covers and runs as two column blocks
        assert _lib.tc_launch_count(1) - dense0 >= 4 * 4 + 2 * 4 * 2
    pointgnn_b200.set_precision('fp32')


def _edge_case(g, scope, mode):
    coords, keypoints, edges = g.graph_tuple()
    rng = np.random.default_rng(5)
    w = g.weights
    if mode == 'pool':
        lc = g.layer_configs[0]
        feats = g.graph['intensity']
        return lc, feats, coords[0], keypoints[0], edges[0]
    lc = [l for l in g.layer_configs if l['scope'] == scope][0]
    k = coords[1].shape[0]
    d = w[scope + '/combined_features/fully_connected_1/weights'].shape[1]
    feats = np.abs(rng.standard_normal((k, d))).astype(np.float32) * 0.3
    return lc, feats, coords[1], keypoints[1], edges[1]


@pytest.mark.parametrize('name', ['car', 'ped'])
@pytest.mark.parametrize('precision', PRECISIONS)
def test_layers_vs_oracle(name, precision, request):
    """PointSetPooling.apply_regular and GraphNetAutoCenter.apply_regular, layer by layer."""
    _need(precision)
    import pointgnn_b200
    from pointgnn_b200.models import gnn
    g = request.getfixturevalue(name)
    pointgnn_b200.set_precision(precision)
    store = gnn.VariableStore(g.weights)
    try:
        lc, feats, xyz, kp, ed = _edge_case(g, 'layer1', 'pool')
        want = ognn.point_set_pooling(g.weights, 'layer1', feats, xyz, kp, ed, **lc['kwargs'])
        with gnn.variable_session(store), gnn.variable_scope('layer1'):
            got = gnn.PointSetPooling().apply_regular(_cuda(feats), _cuda(xyz), _cuda(kp, torch.int32),
                                                      _cuda(ed, torch.int32), **lc['kwargs'])
        assert got.shape == want.shape and np.abs(got.cpu().numpy() - want).max() < TOL
        for scope in ('layer2', 'layer4'):
            lc, feats, xyz, kp, ed = _edge_case(g, scope, 'gnn')
            want = ognn.graph_net_auto_center(g.weights, scope, feats, xyz, kp, ed, **lc['kwargs'])
            with gnn.variable_session(store), gnn.variable_scope(scope):
                got = gnn.GraphNetAutoCenter().apply_regular(_cuda(feats), _cuda(xyz), None, _cuda(ed, torch.int32),
                                                             **lc['kwargs'])
            err = np.abs(got.cpu().numpy() - want).max()
            assert err < TOL, (scope, err)
            # auto_offset=False path (configs/car_fixed_T3_train_config:64)
            kw = dict(lc['kwargs'], auto_offset=False)
            want = ognn.graph_net_auto_center(g.weights, scope, feats, xyz, kp, ed, **kw)
            with gnn.variable_session(store), gnn.variable_scope(scope):
                # the un-offset layer does not create the offset MLP variables, scope counters differ
                got = gnn.GraphNetAutoCenter().apply_regular(_cuda(feats), _cuda(xyz), None, _cuda(ed, torch.int32), **kw)
            assert np.abs(got.cpu().numpy() - want).max() < TOL
    finally:
        pointgnn_b200.set_precision('fp32')


def test_fused_equals_op_by_op(car):
    """Custom plugin functions take the op-by-op route; results must equal the fused kernel."""
    from pointgnn_b200.models import gnn

    def my_mlp(features, Ks, is_logits, normalization_type, activation_type):
        return gnn.multi_layer_neural_network_fn(features, Ks, is_logits, normalization_type, activation_type)

    def my_max(f, c, n):
        return gnn.graph_scatter_max_fn(f, c, n)

    store = gnn.VariableStore(car.weights)
    lc, feats, xyz, kp, ed = _edge_case(car, 'layer3', 'gnn')
    args = (_cuda(feats), _cuda(xyz), None, _cuda(ed, torch.int32))
    with gnn.variable_session(store), gnn.variable_scope('layer3'):
        fused = gnn.GraphNetAutoCenter().apply_regular(*args, **lc['kwargs'])
    with gnn.variable_session(store), gnn.variable_scope('layer3'):
        plain = gnn.GraphNetAutoCenter(edge_feature_fn=my_mlp, aggregation_fn=my_max, update_fn=my_mlp,
                                       auto_offset_fn=my_mlp).apply_regular(*args, **lc['kwargs'])
    assert np.abs(fused.cpu().numpy() - plain.cpu().numpy()).max() < 1e-4
    lc, feats, xyz, kp, ed = _edge_case(car, 'layer1', 'pool')
    args = (_cuda(feats), _cuda(xyz), _cuda(kp, torch.int32), _cuda(ed, torch.int32))
    with gnn.variable_session(store), gnn.variable_scope('layer1'):
        fused = gnn.PointSetPooling().apply_regular(*args, **lc['kwargs'])
    with gnn.variable_session(store), gnn.variable_scope('layer1'):
        plain = gnn.PointSetPooling(point_feature_fn=my_mlp, aggregation_fn=my_max,
                                    output_fn=my_mlp).apply_regular(*args, **lc['kwargs'])
    assert np.abs(fused.cpu().numpy() - plain.cpu().numpy()).max() < 1e-4


def _predict(g, layer_configs, precision, inputs):
    import pointgnn_b200
    from pointgnn_b200.models import models
    pointgnn_b200.set_precision(precision)
    try:
        model = models.get_model(g.config['model_name'])(
            num_classes=g.config['num_classes'], box_encoding_len=7, mode='test',
            **dict(g.config['model_kwargs'], layer_configs=layer_configs))
        model.load_weights(g.weights)
        logits, boxes = model.predict(*inputs, is_training=True)       # run.py:254 feeds True
        probs = model.postprocess(logits)
    finally:
        pointgnn_b200.set_precision('fp32')
    return logits, boxes, probs


@pytest.mark.parametrize('name', ['car', 'ped'])
@pytest.mark.parametrize('precision', PRECISIONS)
def test_predict_matches_golden(name, precision, request):
    """Whole model (pool + 3 GNN iterations + predictor) on the pinned graph vs the golden logits."""
    _need(precision)
    g = request.getfixturevalue(name)
    coords, keypoints, edges = g.graph_tuple()
    from pointgnn_b200 import _lib
    tc0 = (_lib.tc_launch_count(0), _lib.tc_launch_count(1))
    logits, boxes, probs = _predict(g, g.layer_configs, precision, (g.graph['intensity'], coords, keypoints, edges))
    if precision == 'bf16x3':
        # the tensor-core kernels must really have run: 3 GNN iterations (+ the car pooling layer) are
        # segment-max tensor-core launches, and the wide per-vertex layers go through the dense tensor-core
        # kernel (no silent FFMA fallback).  The ped pooling MLP (4 -> 32 -> 64 -> 128 -> 256 -> 512) ends in two
        # segment-max launches: its last layer (256 -> 512) runs as two column blocks of 256.
        assert _lib.tc_launch_count(0) - tc0[0] == (4 if name == 'car' else 5)
        assert _lib.tc_launch_count(1) - tc0[1] >= 10
    assert isinstance(logits, np.ndarray) and logits.shape == g.gnn['logits'].shape
    assert boxes.shape == g.gnn['boxes'].shape
    assert np.abs(logits - g.gnn['logits']).max() < TOL
    assert np.abs(boxes - g.gnn['boxes']).max() < TOL
    assert np.abs(probs - ognn.postprocess(g.gnn['logits'])).max() < 1e-4
    assert np.array_equal(probs.argmax(1), ognn.postprocess(g.gnn['logits']).argmax(1))


@pytest.mark.parametrize('name', ALL_CHECKPOINTS)
@pytest.mark.parametrize('precision', PRECISIONS)
def test_every_checkpoint_matches_the_reference_graph(name, precision):
    """All seven shipped checkpoints (T0..T3, trainval, car_fixed = auto_offset False, ped_cyl) against
    tests/golden/gnn_<cfg>.npz = the outputs of the reference's own saved TensorFlow graph
    (checkpoints/<cfg>/model-N.meta interpreted by oracle/graphdef.py): logits, box encodings, class
    probabilities within the 1e-3 budget of north_star."""
    _need(precision)
    g = load_golden(name)
    coords, keypoints, edges = g.graph_tuple()
    logits, boxes, probs = _predict(g, g.layer_configs, precision, (g.graph['intensity'], coords, keypoints, edges))
    assert logits.shape == g.gnn['logits'].shape and boxes.shape == g.gnn['boxes'].shape
    assert np.abs(logits - g.gnn['logits']).max() < TOL, name
    assert np.abs(boxes - g.gnn['boxes']).max() < TOL, name
    assert np.abs(probs - g.gnn['probs']).max() < 1e-4, name


# (checkpoint, points per frame, full 360, frames batched, precisions): the BASELINE.json configurations at
# FULL size, checked against the CPU oracle port (oracle/cpu_reference.predict, itself checked against
# oracle/gnn.py and so against the reference's saved graph in the CPU suite)
FULL_SIZE = [
    ('car_auto_T3_train', 20000, False, 1, ('fp32', 'bf16x3')),       # C2
    ('car_auto_T3_train', 120000, True, 1, ('bf16x3',)),              # C3
    ('ped_cyl_auto_T3_trainval', 20000, False, 8, ('bf16x3',)),       # C4: batch of 8 (batch_data layout)
    ('car_auto_T0_train', 20000, False, 1, ('bf16x3',)),
    ('car_auto_T2_train', 20000, False, 1, ('bf16x3',)),
    ('car_fixed_T3_train', 20000, False, 1, ('bf16x3',)),
]


@pytest.mark.parametrize('name,num_points,full_360,frames,precisions', FULL_SIZE,
                         ids=['C2_car_T3_20k', 'C3_car_T3_120k', 'C4_ped_b8', 'car_T0_20k', 'car_T2_20k', 'car_fixed_20k'])
def test_full_size_vs_oracle(name, num_points, full_360, frames, precisions):
    """CUDA vs the oracle at BASELINE sizes: the graph is built on the GPU (edge lists of the first frame are
    compared with the oracle's graph builder bit-exactly), the forward pass runs on the GPU and on the CPU
    oracle from the SAME vertex / edge arrays, outputs within 1e-3."""
    from oracle import cpu_reference
    from pointgnn_b200.models import graph_gen
    g = load_golden(name)
    clouds = [synth.lidar_frame(70 + i, num_points, full_360) for i in range(frames)]
    xyz = np.vstack([c[0] for c in clouds])
    inten = np.vstack([c[1] for c in clouds])
    fp = np.arange(frames + 1, dtype=np.int32) * num_points
    coords, kp, edges = graph_gen.gen_multi_level_local_graph_v3(xyz, frame_ptr=fp, **g.graph_kwargs)
    if num_points <= 20000:
        co, ko, eo = ograph.gen_multi_level_local_graph_v3(clouds[0][0], **g.graph_kwargs)
        k0, (n0, n1) = len(ko[0]), (len(eo[0]), len(eo[1]))
        assert np.array_equal(kp[0][:k0], ko[0])
        assert np.array_equal(edges[0][:n0], eo[0]) and np.array_equal(edges[1][:n1], eo[1])
    want_l, want_b, want_p = cpu_reference.predict(g.weights, g.layer_configs, g.config['num_classes'], 7, inten,
                                                   coords, kp, edges)
    for precision in precisions:
        _need(precision)
        logits, boxes, probs = _predict(g, g.layer_configs, precision, (inten, coords, kp, edges))
        err = max(np.abs(logits - want_l).max(), np.abs(boxes - want_b).max())
        assert err < TOL, (name, precision, err)
        assert np.abs(probs - want_p).max() < 1e-4


@pytest.mark.parametrize('precision', PRECISIONS)
def test_car_auto_T1_end_to_end(car, precision):
    """BASELINE config 1: car_auto_T1 (pool + 1 GNN iteration + predictor), graph built on the GPU,
    20k-point synthetic cloud, vs the CPU oracle on the oracle's own graph."""
    _need(precision)
    from pointgnn_b200.models import graph_gen
    t1_layers = car.layer_configs[:2] + car.layer_configs[-1:]
    xyz, intensity = synth.lidar_frame(0, 20000)
    graph_np = graph_gen.get_graph_generate_fn('multi_level_local_graph_v3')(xyz, **car.graph_kwargs)
    co, kp, ed = ograph.gen_multi_level_local_graph_v3(xyz, **car.graph_kwargs)
    for a, b in zip(graph_np[2], ed):
        assert np.array_equal(a, b)
    logits, boxes, _ = _predict(car, t1_layers, precision, (intensity,) + tuple(graph_np))
    want_l, want_b = ognn.predict(car.weights, t1_layers, 4, 7, intensity, co, kp, ed)
    assert np.abs(logits - want_l).max() < TOL and np.abs(boxes - want_b).max() < TOL


def test_device_resident_predict_and_batch(car):
    """CUDA-tensor inputs stay on the device; a 2-frame batch (batch_data layout) equals per-frame results."""
    from pointgnn_b200.models import graph_gen
    clouds = [synth.lidar_frame(i, 4000) for i in (30, 31)]
    xyz = torch.from_numpy(np.vstack([c[0] for c in clouds])).cuda()
    inten = torch.from_numpy(np.vstack([c[1] for c in clouds])).cuda()
    fp = torch.tensor([0, 4000, 8000], dtype=torch.int32, device='cuda')
    coords, kp, edges, fps = graph_gen.gen_multi_level_local_graph_v3(xyz, frame_ptr=fp, return_frame_ptr=True,
                                                                     **car.graph_kwargs)
    logits, boxes, _ = _predict(car, car.layer_configs, 'fp32', (inten, coords, kp, edges))
    assert logits.is_cuda and boxes.is_cuda
    k0 = int(fps[1][1])
    for i, (c, it) in enumerate(clouds):
        g1 = graph_gen.gen_multi_level_local_graph_v3(c, **car.graph_kwargs)
        l1, b1, _ = _predict(car, car.layer_configs, 'fp32', (it,) + tuple(g1))
        sl = slice(0, k0) if i == 0 else slice(k0, None)
        assert np.abs(logits[sl].cpu().numpy() - l1).max() < 1e-4
        assert np.abs(boxes[sl].cpu().numpy() - b1).max() < 1e-4


@pytest.mark.parametrize('precision', PRECISIONS)
def test_full_size_properties(car, precision):
    """BASELINE config sizes (20 000-point frames, ~490 k edges per frame, thousands of tiles, segments that
    straddle tiles and CTA pairs), checked through size-independent properties instead of the slow oracle:
    * batch invariance: a 3-frame batch (batch_data layout) == the three single-frame results,
    * precision agreement: the tensor-core path == the fp32 FFMA path within the 1e-3 budget,
    * aggregation identity: the fused gather/MLP/segment-max layer == the op-by-op composition
      (gather_rows -> fully_connected -> scatter_max) of the same layer on the same edges."""
    import pointgnn_b200
    from pointgnn_b200 import _lib
    from pointgnn_b200.models import gnn, graph_gen
    clouds = [synth.lidar_frame(i, 20000) for i in (40, 41, 42)]
    xyz = torch.from_numpy(np.vstack([c[0] for c in clouds])).cuda()
    inten = torch.from_numpy(np.vstack([c[1] for c in clouds])).cuda()
    fp = torch.tensor([0, 20000, 40000, 60000], dtype=torch.int32, device='cuda')
    coords, kp, edges, fps = graph_gen.gen_multi_level_local_graph_v3(xyz, frame_ptr=fp, return_frame_ptr=True,
                                                                     **car.graph_kwargs)
    assert edges[1].shape[0] > 1_000_000
    logits, boxes, _ = _predict(car, car.layer_configs, precision, (inten, coords, kp, edges))
    ref_l, ref_b, _ = _predict(car, car.layer_configs, 'fp32', (inten, coords, kp, edges))
    assert float((logits - ref_l).abs().max()) < 1e-3 and float((boxes - ref_b).abs().max()) < 1e-3
    bounds = [int(v) for v in fps[1].cpu()]
    for i, (c, it) in enumerate(clouds):
        g1 = graph_gen.gen_multi_level_local_graph_v3(torch.from_numpy(c).cuda(), **car.graph_kwargs)
        l1, b1, _ = _predict(car, car.layer_configs, precision, (torch.from_numpy(it).cuda(),) + tuple(g1))
        sl = slice(bounds[i], bounds[i + 1])
        assert l1.shape[0] == bounds[i + 1] - bounds[i]
        assert float((logits[sl] - l1).abs().max()) < 2e-4
        assert float((boxes[sl] - b1).abs().max()) < 2e-4
    # fused layer == op-by-op composition on the full-size keypoint graph (layer 2 weights)
    pointgnn_b200.set_precision(precision)
    k = coords[1].shape[0]
    feats = torch.rand((k, 300), device='cuda') * 0.5
    sc = 'layer2/extract_vertex_features/fully_connected'
    ws = [torch.from_numpy(car.weights[sc + '/weights']).cuda(), torch.from_numpy(car.weights[sc + '_1/weights']).cuda()]
    bs = [torch.from_numpy(car.weights[sc + '/biases']).cuda(), torch.from_numpy(car.weights[sc + '_1/biases']).cuda()]
    src, dst = edges[1][:, 0].contiguous(), edges[1][:, 1].contiguous()
    fused = _lib.edge_mlp_max(1, feats, coords[1], coords[1], None, src, dst, k, ws, bs,
                              precision=pointgnn_b200.get_precision())
    e0 = 400_000                                   # a prefix of the edge list keeps the [E, 303] tensor small
    d_last = int(dst[e0 - 1])
    e0 = int((dst <= d_last).sum())                # whole destination segments only
    x = torch.cat([_lib.gather_rows(feats, src[:e0]),
                   _lib.gather_rows(coords[1], src[:e0]) - _lib.gather_rows(coords[1], dst[:e0])], dim=1).contiguous()
    h = _lib.fully_connected(x, ws[0], bs[0], True, precision=0)
    h = _lib.fully_connected(h, ws[1], bs[1], True, precision=0)
    ref = _lib.scatter_max(h, dst[:e0], d_last + 1)
    assert float((fused[:d_last + 1] - ref).abs().max()) < 2e-4
    pointgnn_b200.set_precision('fp32')


def test_errors_are_python_exceptions(car):
    from pointgnn_b200 import _lib
    from pointgnn_b200.models import gnn, models
    m = models.get_model('multi_layer_fast_local_graph_model_v2')(num_classes=4, box_encoding_len=7, mode='test',
                                                                  **car.config['model_kwargs'])
    with pytest.raises(RuntimeError):
        m.predict(np.zeros((1, 1), np.float32), [], [], [])
    # out-of-range edge index (TF: InvalidArgumentError at sess.run)
    w = torch.zeros((4, 8), device='cuda')
    b = torch.zeros(8, device='cuda')
    f = torch.zeros((5, 1), device='cuda')
    x = torch.zeros((5, 3), device='cuda')
    src = torch.tensor([0, 9], dtype=torch.int32, device='cuda')
    dst = torch.tensor([0, 0], dtype=torch.int32, device='cuda')
    with pytest.raises(_lib.PointGNNError):
        _lib.edge_mlp_max(1, f, x, x, None, src, dst, 5, [w], [b])
    with pytest.raises(ValueError):
        _lib.fully_connected(torch.zeros((2, 3), device='cuda'), w, b, True)
    store = gnn.VariableStore({})
    with gnn.variable_session(store), gnn.variable_scope('layer9'):
        with pytest.raises(KeyError):
            gnn.multi_layer_neural_network_fn(torch.zeros((2, 3), device='cuda'), Ks=(4,), normalization_type='NONE')
    with pytest.raises(NotImplementedError):
        gnn.multi_layer_neural_network_fn(torch.zeros((2, 3), device='cuda'), Ks=(4,))   # default BN: not built
    with pytest.raises(ValueError):     # residual of the wrong shape (the reference's tf.add raises)
        _lib.fully_connected(torch.zeros((2, 4), device='cuda'), w, b, True, residual=torch.zeros((2, 3), device='cuda'))


def test_index_contract_of_predict(car):
    """The trusted-index fast path must not read out of bounds on inconsistent inputs (TF raises
    InvalidArgumentError at sess.run for each of these): feature / keypoint tensors whose row counts do not
    match the coordinate lists, keypoint indices out of range, and graph_gen edge tensors edited in place."""
    from pointgnn_b200 import _lib
    from pointgnn_b200.models import graph_gen, models
    m = models.get_model('multi_layer_fast_local_graph_model_v2')(num_classes=4, box_encoding_len=7, mode='test',
                                                                  **car.config['model_kwargs'])
    m.load_weights(car.weights)
    xyz, inten = synth.lidar_frame(5, 2000)
    xyz_t, inten_t = torch.from_numpy(xyz).cuda(), torch.from_numpy(inten).cuda()
    coords, kp, edges = graph_gen.gen_multi_level_local_graph_v3(xyz_t, **car.graph_kwargs)
    good_l, _ = m.predict(inten_t, coords, kp, edges)
    with pytest.raises(ValueError):
        m.predict(inten_t[:-1], coords, kp, edges)                       # features shorter than coords[0]
    with pytest.raises(ValueError):
        m.predict(inten_t, coords, [kp[0][:-1], kp[1]], edges)           # keypoints shorter than coords[1]
    bad_kp = kp[0].clone()
    bad_kp[0, 0] = xyz.shape[0] + 7
    with pytest.raises(_lib.PointGNNError):
        m.predict(inten_t, coords, [bad_kp, kp[1]], edges)               # keypoint index out of range
    edited = edges[1]
    edited[:, 0] += coords[1].shape[0]                                   # in-place edit keeps the attribute ...
    with pytest.raises(_lib.PointGNNError):                              # ... but the version stamp differs
        m.predict(inten_t, coords, kp, [edges[0], edited])
    edited[:, 0] -= coords[1].shape[0]
    again_l, _ = m.predict(inten_t, coords, kp, [edges[0], edited])      # re-checked, in range again
    assert torch.equal(good_l, again_l)


@pytest.mark.parametrize('d,c_in', [(300, 300), (256, 256), (64, 32), (128, 300)])
def test_tc_edge_kernel_shapes_and_tails(d, c_in):
    """The tensor-core edge kernel on its own: odd widths, tails, tiny / huge / empty segments."""
    _need('bf16x3')
    from pointgnn_b200 import _lib
    rng = np.random.default_rng(d)
    nv = 700
    for case, (e, pattern) in enumerate(((1, 'one'), (255, 'long'), (256, 'long'), (257, 'short'), (5000, 'mixed'),
                                         (33000, 'mixed'))):
        if pattern == 'one':
            dst = np.array([3])
        elif pattern == 'long':
            dst = np.sort(rng.integers(0, 3, e))                      # segments spanning tiles
        elif pattern == 'short':
            dst = np.sort(rng.integers(0, nv, e))                     # ~1 edge per segment, many empty
        else:
            dst = np.sort(np.concatenate([rng.integers(0, nv, e // 2), rng.integers(10, 14, e - e // 2)]))
        src = rng.integers(0, nv, e)
        f = (rng.standard_normal((nv, c_in)) * 0.5).astype(np.float32)
        x = (rng.standard_normal((nv, 3)) * 20).astype(np.float32)
        xd = x + (rng.standard_normal((nv, 3)) * 0.1).astype(np.float32)
        w1 = (rng.standard_normal((c_in + 3, d)) / np.sqrt(c_in)).astype(np.float32)
        b1 = (rng.standard_normal(d) * 0.1).astype(np.float32)
        w2 = (rng.standard_normal((d, d)) / np.sqrt(d)).astype(np.float32)
        b2 = (rng.standard_normal(d) * 0.1).astype(np.float32)
        e0 = np.concatenate([f[src], x[src] - xd[dst]], axis=1)
        h = np.maximum(np.maximum(e0 @ w1 + b1, 0) @ w2 + b2, 0)
        want = ognn.graph_scatter_max_fn(h, dst, nv)
        for prec in (0, 1):
            before = _lib.tc_launch_count(0)
            got = _lib.edge_mlp_max(1, _cuda(f), _cuda(x), _cuda(xd), None, _cuda(src.astype(np.int32)),
                                    _cuda(dst.astype(np.int32)), nv, [_cuda(w1), _cuda(w2)], [_cuda(b1), _cuda(b2)],
                                    precision=prec).cpu().numpy()
            assert _lib.tc_launch_count(0) - before == (1 if prec == 1 else 0), (d, prec)
            empty = want == np.finfo(np.float32).min
            assert np.array_equal(got == np.finfo(np.float32).min, empty), (case, prec)
            err = np.abs(got - want)[~empty].max() if (~empty).any() else 0.0
            assert err < (2e-4 if prec == 0 else 1e-3), (d, case, prec, err)


@pytest.mark.parametrize('dims', [(4, 32, 64, 128, 300), (4, 32, 64, 128, 256, 512), (4, 32, 64, 128, 256, 300),
                                  (4, 16, 64, 200), (4, 32, 128, 64)])
def test_tc_pool_chain_shapes_and_tails(dims):
    """The point-set pooling MLP on tensor cores: per-edge layers in store mode, then the segment-max layer (car
    shape; ped shape 256 -> 512 as two column blocks; a last layer of 300 in one block), tails, one-edge /
    tile-spanning / empty segments, keypoint indirection."""
    _need('bf16x3')
    from pointgnn_b200 import _lib
    rng = np.random.default_rng(sum(dims))
    nv, nk = 900, 400
    launches = -(-dims[-1] // 304)           # one segment-max launch per column block of at most 304 features
    ws = [(rng.standard_normal((dims[i], dims[i + 1])) / np.sqrt(dims[i])).astype(np.float32) for i in range(len(dims) - 1)]
    bs = [(rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32) for i in range(len(dims) - 1)]
    for case, (e, pattern) in enumerate(((1, 'one'), (255, 'long'), (256, 'long'), (257, 'short'), (5000, 'mixed'),
                                         (70000, 'mixed'))):
        if pattern == 'one':
            dst = np.array([3])
        elif pattern == 'long':
            dst = np.sort(rng.integers(0, 3, e))
        elif pattern == 'short':
            dst = np.sort(rng.integers(0, nk, e))
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
        before = _lib.tc_launch_count(0)
        got = _lib.edge_mlp_max(0, _cuda(f), _cuda(x), _cuda(x), _cuda(kp.astype(np.int32)), _cuda(src.astype(np.int32)),
                                _cuda(dst.astype(np.int32)), nk, [_cuda(w) for w in ws], [_cuda(b) for b in bs],
                                precision=1).cpu().numpy()
        assert _lib.tc_launch_count(0) - before == launches, (dims, case)
        empty = want == np.finfo(np.float32).min
        assert np.array_equal(got == np.finfo(np.float32).min, empty), (dims, case)
        scale = max(1.0, float(np.abs(want[~empty]).max())) if (~empty).any() else 1.0
        err = np.abs(got - want)[~empty].max() if (~empty).any() else 0.0
        assert err < 1e-3 * scale, (dims, case, err, scale)


def test_scatter_sum_and_mean_vs_numpy(car):
    """graph_scatter_sum_fn / graph_scatter_mean_fn (gnn.py:111-119: unsorted_segment_sum / _mean; no shipped config
    selects them) against NumPy, sorted and unsorted ids, empty segments -> 0; and as the aggregation plug-in of a
    pooling layer (op-by-op path) against the same composition in NumPy."""
    from pointgnn_b200.models import gnn
    rng = np.random.default_rng(3)
    for e, k, c, sort in ((1, 3, 1, True), (5000, 300, 300, True), (7001, 41, 19, False), (260, 9000, 64, True)):
        feats = rng.standard_normal((e, c)).astype(np.float32)
        ids = rng.integers(0, k, e)
        if sort:
            ids = np.sort(ids)
        want = np.zeros((k, c), np.float64)
        np.add.at(want, ids, feats.astype(np.float64))
        cnt = np.bincount(ids, minlength=k).astype(np.float64)
        got = gnn.graph_scatter_sum_fn(_cuda(feats), _cuda(ids.astype(np.int32)), k).cpu().numpy()
        assert got.shape == (k, c) and np.abs(got - want).max() < 1e-4 * max(1.0, np.abs(want).max())
        gotm = gnn.graph_scatter_mean_fn(_cuda(feats), _cuda(ids.astype(np.int32)), k).cpu().numpy()
        wantm = want / np.maximum(cnt, 1.0)[:, None]
        assert np.abs(gotm - wantm).max() < 1e-5 * max(1.0, np.abs(wantm).max())
        assert np.all(gotm[cnt == 0] == 0.0) and np.all(got[cnt == 0] == 0.0)
    # as a layer plug-in
    lc, feats, xyz, kp, ed = _edge_case(car, 'layer1', 'pool')
    store = gnn.VariableStore(car.weights)
    with gnn.variable_session(store), gnn.variable_scope('layer1'):
        got = gnn.PointSetPooling(aggregation_fn=gnn.graph_scatter_mean_fn).apply_regular(
            _cuda(feats), _cuda(xyz), _cuda(kp, torch.int32), _cuda(ed, torch.int32), **lc['kwargs']).cpu().numpy()
    w = car.weights
    src, dst = ed[:, 0], ed[:, 1]
    h = np.concatenate([feats[src], xyz[src] - xyz[kp[dst, 0]]], axis=1).astype(np.float64)
    names = ['layer1/extract_vertex_features/fully_connected' + s for s in ('', '_1', '_2', '_3')]
    for n in names:
        h = np.maximum(h @ w[n + '/weights'] + w[n + '/biases'], 0)
    agg = np.zeros((len(kp), h.shape[1]))
    np.add.at(agg, dst, h)
    agg /= np.maximum(np.bincount(dst, minlength=len(kp)), 1)[:, None]
    for n in ('layer1/combined_features/fully_connected', 'layer1/combined_features/fully_connected_1'):
        agg = np.maximum(agg @ w[n + '/weights'] + w[n + '/biases'], 0)
    assert np.abs(got - agg).max() < 1e-3 * max(1.0, np.abs(agg).max())


# edge layer shapes: (mode, feature channels, layer widths) - a GNN iteration (two layers) and a pooling MLP (three)
EDGE_SHAPES = {'gnn': (1, 32, (64, 64)), 'pool': (0, 1, (32, 64, 128))}


def _edge_layer_inputs(shape, seed):
    """Random weights and a destination-sorted edge list for one EDGE_SHAPES entry."""
    from pointgnn_b200 import _lib
    mode, c_in, widths = EDGE_SHAPES[shape]
    rng = np.random.default_rng(seed)
    nv, e = 700, 3000
    dims = [c_in + 3] + list(widths)
    ws = [_cuda((rng.standard_normal((dims[i], dims[i + 1])) / np.sqrt(dims[i])).astype(np.float32))
          for i in range(len(widths))]
    bs = [_cuda((rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32)) for i in range(len(widths))]
    f = _cuda((rng.standard_normal((nv, c_in)) * 0.5).astype(np.float32))
    x = _cuda((rng.standard_normal((nv, 3)) * 20).astype(np.float32))
    if mode == 1:      # GNN: the destinations are the vertices, xyz_dst the offset coordinates
        nd, xd, kp = nv, x + _cuda((rng.standard_normal((nv, 3)) * 0.1).astype(np.float32)), None
    else:              # pooling: the destinations are keypoints, indirected into xyz_dst
        nd, xd = 300, x
        kp = _cuda(rng.integers(0, nv, nd).astype(np.int32))
    src = _cuda(rng.integers(0, nv, e).astype(np.int32))
    dst = _cuda(np.sort(rng.integers(0, nd, e)).astype(np.int32))
    kind = _lib.PG_LAYER_EDGE_GNN if mode == 1 else _lib.PG_LAYER_EDGE_POOL
    return mode, kind, dims, ws, bs, (f, x, xd, kp), src, dst, nd


def _counted(fn):
    """fn() and the number of kernel launches it made."""
    from pointgnn_b200 import _lib
    before = _lib.launch_count()
    out = fn()
    return out, _lib.launch_count() - before


@pytest.mark.parametrize('precision', [0, 1])
def test_per_call_equals_prepared(precision):
    """pg_fully_connected / pg_edge_mlp_max equal pg_layer_create + pg_layer_mlp / pg_layer_edge_mlp_max bit for bit
    and launch as many kernels (the segment max is an exact max, so the order of its atomics does not matter)."""
    if precision == 1:
        _need('bf16x3')
    from pointgnn_b200 import _lib
    rng = np.random.default_rng(12)
    # 600 features run as two column blocks on the tensor cores
    for m, k, n in ((1000, 300, 300), (513, 4, 32), (257, 300, 600)):
        x = _cuda(rng.standard_normal((m, k)).astype(np.float32))
        w = _cuda((rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32))
        b = _cuda(rng.standard_normal(n).astype(np.float32))
        r = _cuda(rng.standard_normal((m, n)).astype(np.float32))
        for relu in (True, False):
            for res in (None, r):
                dense0 = _lib.tc_launch_count(1)
                per, per_launches = _counted(
                    lambda: _lib.fully_connected(x, w, b, relu, residual=res, precision=precision))
                if precision == 1 and n == 600:
                    assert _lib.tc_launch_count(1) - dense0 == 2
                layer, create_launches = _counted(
                    lambda: _lib.PreparedLayer(_lib.PG_LAYER_MLP, [w], [b], [k, n], precision))
                prep, apply_launches = _counted(lambda: layer.mlp(x, last_linear=not relu, residual=res))
                assert torch.equal(per, prep), (m, k, n, relu, res is not None)
                assert per_launches == create_launches + apply_launches, (m, k, n, relu, res is not None)
    for shape in EDGE_SHAPES:
        mode, kind, dims, ws, bs, (f, x, xd, kp), src, dst, nd = _edge_layer_inputs(shape, 13)
        per, per_launches = _counted(
            lambda: _lib.edge_mlp_max(mode, f, x, xd, kp, src, dst, nd, ws, bs, precision=precision))
        layer, create_launches = _counted(lambda: _lib.PreparedLayer(kind, ws, bs, dims, precision))
        prep, apply_launches = _counted(lambda: layer.edge_mlp_max(f, x, xd, kp, src, dst, nd))
        assert torch.equal(per, prep), shape
        assert per_launches == create_launches + apply_launches, shape


@pytest.mark.parametrize('shape', list(EDGE_SHAPES))
@pytest.mark.parametrize('precision', [0, 1])
@pytest.mark.parametrize('route', ['per_call', 'prepared'])
def test_edge_index_errors_on_every_route(route, precision, shape):
    """An out-of-range src or dst raises on every edge route, and a trusted call (no read-back) does not stop a
    later untrusted call on the same thread from checking its indices."""
    if precision == 1:
        _need('bf16x3')
    from pointgnn_b200 import _lib
    mode, kind, dims, ws, bs, (f, x, xd, kp), src, dst, nd = _edge_layer_inputs(shape, 14)
    if route == 'prepared':
        layer = _lib.PreparedLayer(kind, ws, bs, dims, precision)

        def call(s, d, trusted=False):
            return layer.edge_mlp_max(f, x, xd, kp, s, d, nd, trusted=trusted)
    else:
        def call(s, d, trusted=False):
            return _lib.edge_mlp_max(mode, f, x, xd, kp, s, d, nd, ws, bs, precision=precision, trusted=trusted)
    good = call(src, dst)
    bad = []
    for pos, value in ((src.numel() // 2, f.shape[0] + 7), (0, -1)):
        s = src.clone()
        s[pos] = value
        bad.append((s, dst))
    for pos, value in ((-1, nd + 3), (0, -1)):          # dst stays non-decreasing
        d = dst.clone()
        d[pos] = value
        bad.append((src, d))
    for s, d in bad:
        with pytest.raises(_lib.PointGNNError, match='out of range'):
            call(s, d)
    assert torch.equal(call(src, dst, trusted=True), good)
    with pytest.raises(_lib.PointGNNError, match='out of range'):
        call(bad[0][0], dst)

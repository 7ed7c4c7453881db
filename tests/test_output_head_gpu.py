"""The class-aware separated predictor and the canonical box codec on the GPU, against the NumPy restatements of
test_output_head_cpu.py (pinned there to the reference's own decoder through tests/golden/box_canonical.npz).

Tolerances.  Separated head: fp32 1e-4 and BF16x3 1e-3 of the restatement, FP16 1e-3 of the FP16 oracle
(tests/fp16_oracle.py) on the zero-padded loc weights, all relative to max(1, |want|).  Whole model: 1e-3 at BF16x3,
the FP16 suite's 8e-3 / 4e-3 at FP16.  Canonical decode: x, y, z and yaw bit for bit (cos / sin are NumPy's float32
routine, restated); the sizes exp(e) l within 4 ulp, because exp is CUDA's expf (within 2 ulp of exp), as in the
all-class rule, whose sizes they equal byte for byte.  NMS: as test_post_stage_gpu.py
(kept sets, labels and indices identical; boxes and scores within 1e-4)."""
import copy
import json
import os
from functools import partial

import numpy as np
import pytest
import torch

import fp16_oracle
from conftest import GOLDEN, Golden
from oracle import gnn as ognn
from oracle import graph as ograph
from oracle import kitti as ok
from oracle import postprocess as opp
from test_activations_cpu import NAMES, activation_oracle
from test_output_head_cpu import (CANONICAL, canonical_decode_all, expanded_weights, separated_checkpoint,
                                  separated_predictor)
from test_run_batched_gpu import _tree

pytestmark = pytest.mark.gpu
BOX = 7
K_SWEEP = (1, 63, 64, 65, 25000)          # around the heads kernel's 64-row tile, and a frame-sized K
WIDTH = {1: 128, 2: 128, 4: 128, 6: 192, 16: 256}    # D per C: multiples of C


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _head_weights(seed, d, c, scope='output'):
    """Seeded separated-predictor variables: cls D -> 64 -> C, loc/cls_c D/C -> 64 -> 64 -> 7."""
    rng = np.random.default_rng(seed)
    w = {}

    def fc(prefix, i, k, n):
        name = prefix + ('/fully_connected' if i == 0 else '/fully_connected_%d' % i)
        w[name + '/weights'] = (rng.standard_normal((k, n)) / np.sqrt(k)).astype(np.float32)
        w[name + '/biases'] = (rng.standard_normal(n) * 0.1).astype(np.float32)

    fc(scope + '/predictor/cls', 0, d, 64)
    fc(scope + '/predictor/cls', 1, 64, c)
    for k in range(c):
        p = scope + '/predictor/loc/cls_%d' % k
        fc(p, 0, d // c, 64)
        fc(p, 1, 64, 64)
        fc(p, 2, 64, BOX)
    return w


def _run_head(weights, features, c, precision, act='ReLU'):
    import pointgnn_b200
    from pointgnn_b200.models import gnn
    pointgnn_b200.set_precision(precision)
    try:
        p = gnn.ClassAwareSeparatedPredictor(cls_fn=partial(gnn.multi_layer_fc_fn, Ks=(64,), num_layer=2),
                                             loc_fn=partial(gnn.multi_layer_fc_fn, Ks=(64, 64), num_layer=3))
        with gnn.variable_session(gnn.VariableStore(weights)), gnn.variable_scope('output'):
            logits, boxes = p.apply_regular(_cuda(features), num_classes=c, box_encoding_len=BOX,
                                            normalization_type='NONE', activation_type=act)
    finally:
        pointgnn_b200.set_precision('fp32')
    return logits.cpu().numpy(), boxes.cpu().numpy()


def _want(weights, features, c, precision, act):
    if precision == 'fp16':
        return fp16_oracle.class_aware_predictor(expanded_weights(weights, 'output', c), 'output', features, c, BOX,
                                                 activation_type=act)
    with activation_oracle():
        return separated_predictor(weights, 'output', features, c, BOX, act)


def _check(got, want, precision, what):
    tol = {'fp32': 1e-4, 'bf16x3': 1e-3, 'fp16': 1e-3}[precision]
    for g, w, name in zip(got, want, ('logits', 'boxes')):
        assert g.shape == w.shape, (what, name, g.shape, w.shape)
        err = float(np.abs(g - w).max())
        assert err <= tol * max(1.0, float(np.abs(w).max())), (what, name, err)


def _precisions():
    from pointgnn_b200 import _lib
    return ['fp32'] + (['bf16x3', 'fp16'] if _lib.tc_available() else [])


@pytest.mark.parametrize('act', NAMES)
@pytest.mark.parametrize('precision', ['fp32', 'bf16x3', 'fp16'])
def test_separated_head_every_activation(precision, act):
    if precision not in _precisions():
        pytest.skip('no wgmma kernels on this device')
    c, d = 4, WIDTH[4]
    w = _head_weights(7, d, c)
    x = np.random.default_rng(8).standard_normal((65, d)).astype(np.float32)
    _check(_run_head(w, x, c, precision, act), _want(w, x, c, precision, act), precision, (precision, act))


@pytest.mark.parametrize('c', sorted(WIDTH))
@pytest.mark.parametrize('precision', ['fp32', 'bf16x3', 'fp16'])
def test_separated_head_classes_and_rows(precision, c):
    if precision not in _precisions():
        pytest.skip('no wgmma kernels on this device')
    d = WIDTH[c]
    w = _head_weights(10 + c, d, c)
    for k in K_SWEEP:
        x = np.random.default_rng(k).standard_normal((k, d)).astype(np.float32)
        _check(_run_head(w, x, c, precision), _want(w, x, c, precision, 'ReLU'), precision, (precision, c, k))


def test_separated_head_indivisible_width_is_an_error_not_a_launch():
    """D = 256, C = 6 (the ped model's shape): predict raises ValueError; pg_layer_create with the flag returns
    PG_ERR_INVALID_ARGUMENT with pg_last_error set.  Nothing is launched."""
    from pointgnn_b200 import _lib
    c, d = 6, 256
    w = _head_weights(3, 252, c)        # 42-row loc weights: no D makes them a valid split of 256
    w['output/predictor/cls/fully_connected/weights'] = np.zeros((d, 64), np.float32)
    launches = _lib.launch_count()
    with pytest.raises(ValueError, match='D = 256.*C = 6'):
        _run_head(w, np.zeros((5, d), np.float32), c, 'fp32')
    names = ['output/predictor/cls/fully_connected', 'output/predictor/cls/fully_connected_1']
    for k in range(c):
        names += ['output/predictor/loc/cls_%d/fully_connected%s' % (k, s) for s in ('', '_1', '_2')]
    ws = [_cuda(w[n + '/weights']) for n in names]
    bs = [_cuda(w[n + '/biases']) for n in names]
    for precision in (0, 1):
        with pytest.raises(_lib.PointGNNError) as err:
            _lib.PreparedLayer(_lib.PG_LAYER_PREDICTOR, ws, bs, [d, 64, c, BOX], precision, separated=True)
        assert err.value.code == _lib.PG_ERR_INVALID_ARGUMENT
        assert 'D = 256' in str(err.value) and 'C = 6' in str(err.value)
    with pytest.raises(_lib.PointGNNError) as err:      # the flag belongs to the predictor only
        _lib.PreparedLayer(_lib.PG_LAYER_MLP, ws[:2], bs[:2], [d, 64, c], 0, separated=True)
    assert err.value.code == _lib.PG_ERR_INVALID_ARGUMENT
    assert _lib.launch_count() == launches


# ---------------------------------------------------------------------------------------------
# whole model: car_auto_T3 with the separated predictor
# ---------------------------------------------------------------------------------------------
def _separated_oracle(config, weights, intensity, coords, keypoints, edges):
    """fp32: oracle/gnn.py's layers up to the predictor (their variables are the shipped ones), then the
    restatement on the last layer's features."""
    shared = copy.deepcopy(config['model_kwargs']['layer_configs'])
    shared[-1]['type'] = 'classaware_predictor'
    c = config['num_classes']
    feats = ognn.predict(expanded_weights(weights, 'output', c), shared, c, BOX, intensity, coords, keypoints, edges,
                         return_features=True)[2][-1]
    return separated_predictor(weights, 'output', feats, c, BOX)


@pytest.mark.parametrize('precision', ['bf16x3', 'fp16'])
def test_separated_car_model_predict(precision):
    import pointgnn_b200
    from pointgnn_b200 import _lib
    from pointgnn_b200.models import models
    if not _lib.tc_available():
        pytest.skip('no wgmma kernels on this device')
    config, weights = separated_checkpoint()
    g = Golden('car_auto_T3_train')
    coords, keypoints, edges = g.graph_tuple()
    intensity = g.graph['intensity']
    c = config['num_classes']
    if precision == 'fp16':
        shared = copy.deepcopy(config['model_kwargs']['layer_configs'])
        shared[-1]['type'] = 'classaware_predictor'
        want_l, want_b = fp16_oracle.predict(expanded_weights(weights, 'output', c), shared, c, BOX, intensity,
                                             coords, keypoints, edges)
        tol_l, tol_b = 8e-3, 4e-3
    else:
        want_l, want_b = _separated_oracle(config, weights, intensity, coords, keypoints, edges)
        tol_l = tol_b = 1e-3
    pointgnn_b200.set_precision(precision)
    try:
        model = models.get_model(config['model_name'])(num_classes=c, box_encoding_len=BOX, mode='test',
                                                       **config['model_kwargs'])
        model.load_weights(weights)
        logits, boxes = model.predict(intensity, coords, keypoints, edges, is_training=True)
    finally:
        pointgnn_b200.set_precision('fp32')
    el, eb = np.abs(logits - want_l).max(), np.abs(boxes - want_b).max()
    print('separated car_auto_T3 %s: %.3g / %.3g' % (precision, el, eb))
    assert el <= tol_l and eb <= tol_b, (precision, el, eb)
    # the separated model really differs from the shipped one
    assert np.abs(boxes - g.gnn['boxes']).max() > 1e-2


# ---------------------------------------------------------------------------------------------
# canonical decoding
# ---------------------------------------------------------------------------------------------
def _ulps(a, b):
    """|a - b| in float32 ulps (ordered-integer distance)."""
    def ordered(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff), i)
    return np.abs(ordered(a) - ordered(b))


def _check_decoded(got, want):
    """x, y, z and yaw bit for bit (NumPy's float32 cos / sin are restated exactly); the sizes exp(e) l within 4 ulp:
    CUDA's expf is within 2 ulp of exp, and the product with l rounds once more."""
    ulps = [int(_ulps(got[..., j], want[..., j]).max()) for j in range(7)]
    assert ulps[0] == ulps[1] == ulps[2] == ulps[6] == 0 and max(ulps[3:6]) <= 4, ulps


@pytest.mark.parametrize('label_method', sorted(opp.LABEL_MAPS))
def test_canonical_decoding_vs_reference_golden(label_method):
    from pointgnn_b200.models import box_encoding
    g = np.load(os.path.join(GOLDEN, 'box_canonical.npz'))
    labels, xyz, enc = g['labels_' + label_method], g['xyz_' + label_method], g['enc_' + label_method]
    want = g['dec_' + label_method]
    fn = box_encoding.get_box_decoding_fn(CANONICAL)
    got = fn(labels, xyz, enc, opp.LABEL_MAPS[label_method])
    assert got.dtype == np.float32 and got.shape == want.shape
    _check_decoded(got, want)
    # the sizes are the all-class rule's, byte for byte
    plain = box_encoding.classaware_all_class_box_decoding(labels, xyz, enc, opp.LABEL_MAPS[label_method])
    assert np.array_equal(got[..., 3:6].view(np.uint32), plain[..., 3:6].view(np.uint32))
    # CUDA tensors in, CUDA tensors out
    got_t = fn(labels, _cuda(xyz), _cuda(enc), opp.LABEL_MAPS[label_method])
    assert got_t.is_cuda and np.array_equal(got_t.cpu().numpy(), got)


def test_decode_boxes_every_pair_with_flag():
    from pointgnn_b200 import _lib
    from pointgnn_b200.models import box_encoding
    g = np.load(os.path.join(GOLDEN, 'box_canonical.npz'))
    enc = np.concatenate([g['enc_yaw'][:, :1], g['enc_yaw'][:, 1:]], axis=1)
    enc = np.tile(enc, (1, 4, 1))                              # [M, 8, 7]: every label of the yaw map
    xyz = g['xyz_yaw']
    table = box_encoding.class_table(opp.LABEL_MAPS['yaw'], 8)
    got = _lib.decode_boxes(_cuda(enc), _cuda(xyz), table, _lib.PG_BOX_CANONICAL).cpu().numpy()
    want = canonical_decode_all(enc, xyz, opp.LABEL_MAPS['yaw'])
    _check_decoded(got, want)
    # without the flag: the all-class rule, the same bytes as the call without the argument
    plain = _lib.decode_boxes(_cuda(enc), _cuda(xyz), table).cpu().numpy()
    assert np.array_equal(_lib.decode_boxes(_cuda(enc), _cuda(xyz), table, 0).cpu().numpy().view(np.uint32),
                          plain.view(np.uint32))
    assert np.abs(plain - opp.decode_boxes(enc, xyz, opp.LABEL_MAPS['yaw'])).max() < 1e-4
    with pytest.raises(_lib.PointGNNError):
        _lib.decode_boxes(_cuda(enc), _cuda(xyz), table, 16)


def _three_frames():
    """Three frames of synthetic network outputs, the middle one without candidates."""
    frames = [opp.synthetic_outputs(71, 10, 20, 4), opp.synthetic_outputs(72, 4, 10, 4),
              opp.synthetic_outputs(73, 12, 25, 4)]
    pts, enc, probs = frames[1]
    probs = np.full_like(probs, 0.25)                   # no class above 1 / C
    frames[1] = (pts, enc, probs)
    fp = np.cumsum([0] + [len(f[0]) for f in frames]).astype(np.int32)
    return frames, fp


@pytest.mark.parametrize('merge,rescore', [(True, True), (False, False)])
def test_postprocess_canonical_three_frames(merge, rescore):
    from pointgnn_b200 import _lib
    from pointgnn_b200.models import box_encoding
    frames, fp = _three_frames()
    pts, enc, probs = (np.vstack([f[i] for f in frames]) for i in range(3))
    table = box_encoding.class_table(opp.LABEL_MAPS['Car'], 4)
    det = _lib.postprocess(_cuda(probs), _cuda(enc), _cuda(pts), _cuda(fp), table, 0.01, merge=merge,
                           rescore=rescore, canonical=True)
    dfp = det['frame_ptr'].cpu().numpy()
    out_l, out_b, out_s, out_i = (det[k].cpu().numpy() for k in ('label', 'box', 'score', 'index'))
    assert dfp[1] < dfp[3] and dfp[2] == dfp[1], dfp            # frame 1 is empty, the others are not
    for f, (p, e, pr) in enumerate(frames):
        sl = slice(dfp[f], dfp[f + 1])
        dec = canonical_decode_all(e, p, opp.LABEL_MAPS['Car'])
        lab, boxes, scores, idx = opp.select_candidates(pr, dec, 4)
        if len(lab) == 0:
            assert dfp[f + 1] == dfp[f]
            continue
        want_l, want_b, want_s, order = opp.nms_boxes_3d_uncertainty(lab, boxes, scores, 0.01, merge, rescore)
        assert np.array_equal(out_i[sl] - fp[f] * 4, idx[order])
        assert np.array_equal(out_l[sl], want_l)
        assert np.abs(out_b[sl] - want_b).max() < 1e-4
        assert np.abs(out_s[sl] - want_s).max() < 1e-4
    # without the flag: the all-class boxes, as detect() without box_encoding_method gives them
    from pointgnn_b200.models import postprocess
    plain = _lib.postprocess(_cuda(probs), _cuda(enc), _cuda(pts), _cuda(fp), table, 0.01, merge=merge,
                             rescore=rescore)
    via_detect = postprocess.detect(_cuda(probs), _cuda(enc), _cuda(pts), _cuda(fp), 'Car', 0.01, merge, rescore)
    for k in ('label', 'box', 'score', 'index', 'frame_ptr'):
        assert np.array_equal(plain[k].cpu().numpy(), via_detect[k].cpu().numpy()), k
    canon = postprocess.detect(_cuda(probs), _cuda(enc), _cuda(pts), _cuda(fp), 'Car', 0.01, merge, rescore,
                               box_encoding_method=CANONICAL)
    assert np.array_equal(canon['box'].cpu().numpy(), out_b)
    assert not np.array_equal(plain['box'].cpu().numpy(), out_b)


# ---------------------------------------------------------------------------------------------
# end to end: run.py with the separated predictor and the canonical codec
# ---------------------------------------------------------------------------------------------
def _e2e_checkpoint(path):
    """The separated car checkpoint with the canonical codec, the object-class logit biases raised by 7 (as in
    test_run_batched_gpu.py, so that the synthetic frames give detections)."""
    os.makedirs(path)
    config, w = separated_checkpoint()
    config['input_features'] = 'i'
    config['box_encoding_method'] = CANONICAL
    b = w['output/predictor/cls/fully_connected_1/biases'].copy()
    b[1:-1] += 7.0
    w['output/predictor/cls/fully_connected_1/biases'] = b
    with open(os.path.join(path, 'config'), 'w') as f:
        json.dump(config, f)
    np.savez(os.path.join(path, 'weights.npz'), **w)
    return config, w


def _oracle_text(root, name, config, weights):
    velo = np.fromfile(os.path.join(root, 'velodyne/testing/velodyne', name + '.bin'), dtype=np.float32).reshape(-1, 4)
    calib = ok.parse_calib(os.path.join(root, 'calib/testing/calib', name + '.txt'))
    xyz, attr = ok.cam_points_in_image(velo, calib, 1242, 375, None)
    coords, kp, edges = ograph.gen_multi_level_local_graph_v3(xyz, **config['runtime_graph_gen_kwargs'])
    logits, boxes = _separated_oracle(config, weights, attr, coords, kp, edges)
    probs = ognn.postprocess(logits)
    last = coords[config['model_kwargs']['layer_configs'][-1]['graph_level'] + 1]
    dec = canonical_decode_all(boxes, last, opp.LABEL_MAPS[config['label_method']])
    lab, bx, sc, idx = opp.select_candidates(probs, dec, config['num_classes'])
    want = []
    if len(lab):
        k_lab, k_box, k_sc, _ = opp.nms_boxes_3d_uncertainty(lab, bx, sc, config['nms_overlapped_thres'])
        want = ok.kitti_labels(k_lab, k_box, k_sc, last[idx // config['num_classes']], calib, config['label_method'])
    return ok.format_kitti(want)


def test_run_separated_canonical_end_to_end(tmp_path):
    from pointgnn_b200 import run
    root = str(tmp_path / 'kitti')
    names = _tree(root)
    ckpt = str(tmp_path / 'ckpt')
    config, weights = _e2e_checkpoint(ckpt)
    out_dir = str(tmp_path / 'out')
    run.main([ckpt, '--test', '--dataset_root_dir', root, '--output_dir', out_dir, '--batch_size', '3'])
    total_rows = 0
    for name in names:
        with open(os.path.join(out_dir, 'data', name + '.txt')) as f:
            got = ok.parse_kitti_text(f.read())
        want = ok.parse_kitti_text(_oracle_text(root, name, config, weights))
        assert len(got) == len(want), (name, len(got), len(want))
        for (n1, v1), (n2, v2) in zip(got, want):
            assert n1 == n2
            assert np.allclose(v1, v2, rtol=2e-3, atol=2e-3), (name, v1, v2)
        total_rows += len(got)
    assert total_rows > 0, 'the synthetic frames produced no row at all: the test would be vacuous'

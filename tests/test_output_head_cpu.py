"""The model's output head beyond the shipped configs: the class-aware separated predictor (gnn.py:165-209) and the
canonical box codec (box_encoding.py:345-395).

NumPy restatements, which the GPU tests (test_output_head_gpu.py) compare against:
  * ``canonical_decode``: classaware_all_class_box_canonical_decoding, float32 in the reference's operation order.  It
    reproduces tests/golden/box_canonical.npz (made from the reference's own function, tools/make_golden.py
    box_canonical) bit for bit.
  * The separated predictor is oracle/gnn.py's ``class_aware_predictor(..., separated=True)``, on real ``np.split``
    slices.  No saved graph of this predictor exists, so that restatement of gnn.py:177-209 is its oracle.
  * ``separated_checkpoint``: the car_auto_T3 weights with each loc head's first weight cut to its slice's rows, the
    checkpoint the end-to-end tests run.
"""
import copy
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import gnn as ognn
from oracle import postprocess as opp

CANONICAL = 'classaware_all_class_box_canonical_encoding'
THREE_ARGUMENT_CODECS = ('direct_encoding', 'center_box_encoding', 'voxelnet_box_encoding',
                         'classaware_voxelnet_box_encoding')


# ---------------------------------------------------------------------------------------------
# restatements
# ---------------------------------------------------------------------------------------------
def canonical_decode(cls_labels, points_xyz, encoded_boxes, label_map):
    """box_encoding.py:345-395: float32 encodings [M, C', 7], labels [M, 1] of slot 0, float32 points [M, 3]."""
    enc = np.asarray(encoded_boxes, dtype=np.float32)
    out = np.copy(enc)
    for name, label in label_map.items():
        if name in ('Background', 'DontCare'):
            continue
        l, h, w = opp.MEDIAN_OBJECT_SIZE[name]
        for lab, a, b, yaw0 in ((label, l, w, None), (label + 1, w, l, 0.5 * np.pi)):
            mask = cls_labels[:, 0] == lab
            yaw = enc[mask, 0, 6] * (np.pi * 0.25)
            out[mask, 0, 0] = enc[mask, 0, 0] * a * np.cos(yaw) + enc[mask, 0, 2] * b * np.sin(yaw)
            out[mask, 0, 1] = enc[mask, 0, 1] * h
            out[mask, 0, 2] = -enc[mask, 0, 0] * a * np.sin(yaw) + enc[mask, 0, 2] * b * np.cos(yaw)
            out[mask, 0, 3] = np.exp(enc[mask, 0, 3]) * l
            out[mask, 0, 4] = np.exp(enc[mask, 0, 4]) * h
            out[mask, 0, 5] = np.exp(enc[mask, 0, 5]) * w
            out[mask, 0, 6] = yaw if yaw0 is None else yaw + yaw0
    out[:, :, :3] = out[:, :, :3] + np.asarray(points_xyz, dtype=np.float32)[:, None, :]
    return out


def canonical_decode_all(box_encodings, points_xyz, label_map):
    """The canonical decoding of every (vertex, class) pair of [K, C, 7] encodings (what pg_decode_boxes computes
    with PG_BOX_CANONICAL): class c of every vertex decoded under label c."""
    k, c, _ = box_encodings.shape
    out = np.empty((k, c, 7), np.float32)
    for cls in range(c):
        labels = np.full((k, 1), cls)
        out[:, cls] = canonical_decode(labels, points_xyz, box_encodings[:, cls:cls + 1], label_map)[:, 0]
    return out


def loc_first_layer(scope_name, c):
    return '%s/predictor/loc/cls_%d/fully_connected/weights' % (scope_name, c)


def expanded_weights(weights, scope_name, num_classes):
    """The separated checkpoint's loc first layers as the [D, H] weights that are zero outside their slice's rows:
    a shared-predictor checkpoint that computes the same function (what PG_FLAG_SEPARATED packs)."""
    out = dict(weights)
    d = weights['%s/predictor/cls/fully_connected/weights' % scope_name].shape[0]
    for c in range(num_classes):
        w = weights[loc_first_layer(scope_name, c)]
        full = np.zeros((d, w.shape[1]), np.float32)
        full[c * w.shape[0]:(c + 1) * w.shape[0]] = w
        out[loc_first_layer(scope_name, c)] = full
    return out


def separated_checkpoint():
    """(config, weights) of car_auto_T3_train with classaware_separated_predictor: loc/cls_c's first weight is rows
    [75 c, 75 c + 75) of the trained one."""
    with open(os.path.join(GOLDEN, 'config_car_auto_T3_train.json')) as f:
        config = json.load(f)
    config = copy.deepcopy(config)
    config['model_kwargs']['layer_configs'][-1]['type'] = 'classaware_separated_predictor'
    weights = dict(np.load(os.path.join(GOLDEN, 'weights_car_auto_T3_train.npz')))
    scope = config['model_kwargs']['layer_configs'][-1]['scope']
    c = config['num_classes']
    for k in range(c):
        w = weights[loc_first_layer(scope, k)]
        s = w.shape[0] // c
        weights[loc_first_layer(scope, k)] = np.ascontiguousarray(w[k * s:(k + 1) * s])
    return config, weights


# ---------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('label_method', sorted(opp.LABEL_MAPS))
def test_canonical_restatement_equals_reference_golden(label_method):
    g = np.load(os.path.join(GOLDEN, 'box_canonical.npz'))
    labels, xyz, enc = g['labels_' + label_method], g['xyz_' + label_method], g['enc_' + label_method]
    label_map = opp.LABEL_MAPS[label_method]
    # the fixture covers every label, far vertices and |e6| up to a few units
    assert set(np.unique(labels)) == set(range(max(label_map.values()) + 1))
    assert np.abs(xyz).max() > 300 and np.abs(enc[:, 0, 6]).max() > 3
    got = canonical_decode(labels, xyz, enc, label_map)
    want = g['dec_' + label_method]
    assert got.dtype == want.dtype == np.float32
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_canonical_restatement_inverts_the_reference_encoder():
    """The reference's canonical encoding (box_encoding.py:301-343), restated in float64, decodes back."""
    rng = np.random.default_rng(5)
    label_map = opp.LABEL_MAPS['yaw']
    labels = rng.choice([1, 2, 3, 4, 5, 6], (400, 1))
    xyz = rng.uniform(-20, 20, (400, 3))
    boxes = np.c_[rng.uniform(-30, 30, (400, 3)), rng.uniform(0.5, 5, (400, 3)), rng.uniform(-1.5, 1.5, 400)]
    enc = boxes.copy()
    for i, lab in enumerate(labels[:, 0]):
        name = [n for n, v in label_map.items() if v in (lab, lab - 1) and n not in ('Background', 'DontCare')][0]
        l, h, w = opp.MEDIAN_OBJECT_SIZE[name]
        x, y, z = boxes[i, :3] - xyz[i]
        yaw = boxes[i, 6] - (0.5 * np.pi if lab != label_map[name] else 0.0)
        a, b = (l, w) if lab == label_map[name] else (w, l)
        enc[i, 0] = (x * np.cos(yaw) - z * np.sin(yaw)) / a
        enc[i, 1] = y / h
        enc[i, 2] = (x * np.sin(yaw) + z * np.cos(yaw)) / b
        enc[i, 3:6] = np.log(boxes[i, 3:6] / np.array([l, h, w]))
        enc[i, 6] = yaw / (np.pi * 0.25)
    dec = canonical_decode(labels, xyz.astype(np.float32), enc[:, None, :].astype(np.float32), label_map)[:, 0]
    assert np.allclose(dec, boxes, rtol=1e-4, atol=1e-4)


def test_box_decoding_names():
    from pointgnn_b200.models import box_encoding, postprocess
    assert box_encoding.get_box_decoding_fn(CANONICAL) is box_encoding.classaware_all_class_box_canonical_decoding
    assert (box_encoding.get_box_decoding_fn('classaware_all_class_box_encoding')
            is box_encoding.classaware_all_class_box_decoding)
    for name in THREE_ARGUMENT_CODECS + ('classaware_all_class_box_encoding', CANONICAL):
        assert box_encoding.get_encoding_len(name) == 7
    for name in THREE_ARGUMENT_CODECS:
        with pytest.raises(KeyError):
            box_encoding.get_box_decoding_fn(name)
        with pytest.raises(ValueError, match=name):
            postprocess.decoding_flags(name)
    with pytest.raises(KeyError):
        box_encoding.get_encoding_len('nope')


@pytest.mark.parametrize('codec', THREE_ARGUMENT_CODECS)
def test_run_rejects_three_argument_codec_before_reading_a_frame(tmp_path, monkeypatch, codec):
    from pointgnn_b200 import run
    ckpt = tmp_path / 'ckpt'
    ckpt.mkdir()
    with open(os.path.join(GOLDEN, 'config_car_auto_T3_train.json')) as f:
        config = json.load(f)
    config['box_encoding_method'] = codec
    (ckpt / 'config').write_text(json.dumps(config))

    def no_dataset(*args, **kwargs):
        raise AssertionError('the dataset was opened')

    monkeypatch.setattr(run, 'KittiDataset', no_dataset)
    with pytest.raises(ValueError, match=codec):
        run.main([str(ckpt), '--test', '--dataset_root_dir', str(tmp_path / 'missing'),
                  '--output_dir', str(tmp_path / 'out')])


def test_header_constants_parse():
    from pointgnn_b200 import _lib
    assert _lib.PG_FLAG_SEPARATED == 0x1000
    assert _lib.PG_BOX_CANONICAL == 8
    # the separated bit is free in the precision word, the codec bit free in pg_postprocess' NMS flags
    assert _lib.PG_FLAG_SEPARATED & (_lib.PG_PRECISION_MASK | _lib.PG_FLAG_TRUSTED_INDICES | _lib.PG_FLAG_ACTIVATION
                                     | _lib.PG_AGG_MASK | _lib.PG_ACT_MASK) == 0
    assert _lib.PG_BOX_CANONICAL & (_lib.PG_NMS_MERGE | _lib.PG_NMS_RESCORE | _lib.PG_NMS_INT_CORNERS) == 0
    _, params = _lib.PROTOTYPES['pg_decode_boxes']
    assert [name for _, name in params][-2:] == ['flags', 'stream']
    from pointgnn_b200.models import box_encoding
    assert box_encoding.DECODING_FLAGS == {'classaware_all_class_box_encoding': 0, CANONICAL: 8}


class _FakeStore(object):
    def __init__(self, weights):
        self.vars = weights
        self.prepared = {}

    def get(self, name):
        return self.vars[name]


class _FakeLayer(object):
    made = []

    def __init__(self, kind, weights, biases, dims, precision, activation, separated=False):
        self.separated = separated
        self.dims = dims
        _FakeLayer.made.append(self)

    def predictor(self, x):
        import torch
        d, h, c, box = self.dims
        m = x.shape[0]
        return torch.zeros((m, c)), torch.zeros((m, c, box)), torch.zeros((m, c))


def test_prepared_cache_keeps_the_predictor_types_apart(monkeypatch):
    """One store, the same variable names: the shared and the separated predictor get their own prepared layer."""
    import torch
    from pointgnn_b200.models import gnn, models
    from pointgnn_b200 import _lib
    monkeypatch.setattr(_lib, 'PreparedLayer', _FakeLayer)
    _FakeLayer.made = []
    config, sep = separated_checkpoint()
    shared = dict(np.load(os.path.join(GOLDEN, 'weights_car_auto_T3_train.npz')))
    store = _FakeStore({k: torch.from_numpy(v) for k, v in shared.items()})
    model = models.get_model('multi_layer_fast_local_graph_model_v2')(
        num_classes=4, box_encoding_len=7, mode='test', **config['model_kwargs'])
    features = torch.zeros((5, 300))
    for kind in ('classaware_predictor', 'classaware_separated_predictor'):
        store.vars.update({k: torch.from_numpy(v) for k, v in (sep if 'separated' in kind else shared).items()})
        with gnn.variable_session(store), gnn.variable_scope('output'):
            model._default_layers_type[kind].apply_regular(features, num_classes=4, box_encoding_len=7,
                                                           normalization_type='NONE')
    assert [layer.separated for layer in _FakeLayer.made] == [False, True]
    assert len(store.prepared) == 2
    assert sorted(key[-1] for key in store.prepared) == [False, True]


def test_separated_predictor_rejects_indivisible_width():
    import torch
    from pointgnn_b200.models import gnn
    from functools import partial
    p = gnn.ClassAwareSeparatedPredictor(cls_fn=partial(gnn.multi_layer_fc_fn, Ks=(64,), num_layer=2),
                                         loc_fn=partial(gnn.multi_layer_fc_fn, Ks=(64, 64), num_layer=3))
    with pytest.raises(ValueError, match=r'D = 256 .* C = 6'):
        p.apply_regular(torch.zeros((3, 256)), num_classes=6, box_encoding_len=7, normalization_type='NONE')


def test_separated_restatement_equals_shared_predictor_on_expanded_weights():
    """gnn.py:196's split is the shared predictor with block-zero loc weights (the identity the kernels use)."""
    config, weights = separated_checkpoint()
    rng = np.random.default_rng(3)
    feats = rng.standard_normal((50, 300)).astype(np.float32)
    logits, boxes = ognn.class_aware_predictor(weights, 'output', feats, 4, 7, separated=True)
    l2, b2 = ognn.class_aware_predictor(expanded_weights(weights, 'output', 4), 'output', feats, 4, 7)
    assert np.allclose(logits, l2, atol=1e-5) and np.allclose(boxes, b2, atol=1e-5)
    assert weights[loc_first_layer('output', 3)].shape == (75, 64)

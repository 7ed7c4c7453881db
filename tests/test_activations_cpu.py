"""Every activation of the reference's table (gnn.py:24-32): ReLU, ReLU6, LeakyReLU, ELU, Sigmoid, Tanh and NONE.

The CPU oracle package implements ReLU, the activation of every shipped config, and stays as it is: the ReLU goldens
pin its structure (concat order, scopes, is_logits handling).  ``activation_oracle()`` runs that same oracle with the
other activations, defined below from TF 1.15's documented behaviour (TF cannot run here and no shipped checkpoint was
trained with them), by substituting its two MLP functions.  The GPU tests compare the kernels against it."""
import contextlib
import copy
import os
import re

import numpy as np
import pytest

from oracle import gnn as ognn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ['NONE', 'ReLU', 'ReLU6', 'LeakyReLU', 'ELU', 'Sigmoid', 'Tanh']


def _elu(x):
    with np.errstate(over='ignore'):
        return np.where(x > 0, x, np.exp(np.minimum(x, 0)) - x.dtype.type(1))


def _sigmoid(x):
    with np.errstate(over='ignore'):
        return x.dtype.type(1) / (x.dtype.type(1) + np.exp(-x))


# tf.nn.relu, relu6, leaky_relu(alpha=0.01) (gnn.py:28), elu (exp(x) - 1 below zero), sigmoid, tanh; None = linear
ACTIVATIONS = {
    'ReLU': lambda x: np.maximum(x, x.dtype.type(0)),
    'ReLU6': lambda x: np.minimum(np.maximum(x, x.dtype.type(0)), x.dtype.type(6)),
    'LeakyReLU': lambda x: np.where(x > 0, x, x.dtype.type(0.01) * x),
    'ELU': _elu,
    'NONE': None,
    'Sigmoid': _sigmoid,
    'Tanh': np.tanh,
}


def activate(name, x):
    fn = ACTIVATIONS[name]
    return x if fn is None else fn(x).astype(x.dtype, copy=False)


def _fc(x, scope, act):
    w, b = scope.next_fc()
    assert x.shape[1] == w.shape[0], (x.shape, w.shape, scope.prefix)
    return activate(act, x @ w.astype(x.dtype) + b.astype(x.dtype)[None, :])


def _mlp(features, scope, Ks=(64, 32, 64), is_logits=False, normalization_type='NONE', activation_type='ReLU'):
    """oracle.gnn.multi_layer_neural_network_fn with any activation (gnn.py:86-104)."""
    assert normalization_type == 'NONE'
    for i in range(len(Ks)):
        last = i == len(Ks) - 1
        features = _fc(features, scope, 'NONE' if (is_logits and last) else activation_type)
        assert features.shape[1] == Ks[i]
    return features


def _fc_fn(sv, scope, Ks=(64, 32, 64), num_classes=4, is_logits=False, num_layer=4, normalization_type='NONE',
           activation_type='ReLU'):
    """oracle.gnn.multi_layer_fc_fn with any activation (gnn.py:34-84)."""
    assert normalization_type == 'NONE' and len(Ks) == num_layer - 1
    features = sv
    for _ in range(num_layer - 1):
        features = _fc(features, scope, activation_type)
    features = _fc(features, scope, 'NONE' if is_logits else activation_type)
    assert features.shape[1] == num_classes
    return features


@contextlib.contextmanager
def activation_oracle():
    """The oracle package with every activation of the table (its layer functions look these names up at call time)."""
    saved = ognn.multi_layer_neural_network_fn, ognn.multi_layer_fc_fn
    ognn.multi_layer_neural_network_fn, ognn.multi_layer_fc_fn = _mlp, _fc_fn
    try:
        yield ognn
    finally:
        ognn.multi_layer_neural_network_fn, ognn.multi_layer_fc_fn = saved


ACTIVATION_KEYS = ('point_MLP_activation_type', 'output_MLP_activation_type', 'edge_MLP_activation_type',
                   'update_MLP_activation_type', 'auto_offset_MLP_feature_activation_type', 'activation_type')


def with_activation(layer_configs, act=None, per_key=None):
    """A copy of layer_configs with every *_activation_type set to act, or each key to per_key[key]."""
    out = copy.deepcopy(layer_configs)
    for lc in out:
        for key in ACTIVATION_KEYS:
            if key in lc['kwargs']:
                lc['kwargs'][key] = act if per_key is None else per_key[key]
    return out


def test_activations_at_chosen_points():
    f = np.float32
    assert activate('ReLU6', np.array([6.5], f))[0] == 6
    assert activate('ReLU6', np.array([-1.0], f))[0] == 0
    assert np.isclose(activate('LeakyReLU', np.array([-2.0], f))[0], -0.02, rtol=1e-6)
    assert np.isclose(activate('ELU', np.array([-1.0], f))[0], np.exp(-1.0) - 1, rtol=1e-6)
    assert activate('Sigmoid', np.array([0.0], f))[0] == 0.5
    assert list(activate('Tanh', np.array([-50.0, 50.0], f))) == [-1, 1]
    x = np.linspace(-9, 9, 101).astype(f)
    assert np.array_equal(activate('NONE', x), x)
    for name in NAMES:
        assert activate(name, x).dtype == np.float32


@pytest.mark.parametrize('name', NAMES)
def test_monotone_non_decreasing(name):
    """What the fused segment max relies on: max_e f(a_e + b) = f(max_e a_e + b)."""
    x = np.concatenate([np.linspace(-100, 100, 400001), np.linspace(-1e-3, 1e-3, 20001), [-3e38, 3e38]])
    y = activate(name, np.sort(x.astype(np.float32)))
    assert not np.isnan(y).any()
    assert (np.diff(y.astype(np.float64)) >= 0).all(), name


@pytest.mark.parametrize('name', ['car', 'ped'])
def test_activation_oracle_with_relu_reproduces_goldens(name, request):
    g = request.getfixturevalue(name)
    coords, keypoints, edges = g.graph_tuple()
    with activation_oracle() as o:
        logits, boxes = o.predict(g.weights, g.layer_configs, g.config['num_classes'], 7, g.graph['intensity'],
                                  coords, keypoints, edges)
    assert np.abs(logits - g.gnn['logits']).max() < 2e-5
    assert np.abs(boxes - g.gnn['boxes']).max() < 2e-5


def test_activation_oracle_runs_every_activation():
    """car_auto_T1 (one GNN iteration) with its own weights, every *_activation_type set to each entry in turn."""
    from conftest import load_golden
    g = load_golden('car_auto_T1_train')
    coords, keypoints, edges = g.graph_tuple()
    outs = {}
    with activation_oracle() as o:
        for name in NAMES:
            lcs = with_activation(g.layer_configs, name)
            logits, boxes = o.predict(g.weights, lcs, g.config['num_classes'], 7, g.graph['intensity'], coords,
                                      keypoints, edges)
            assert logits.dtype == np.float32 and np.isfinite(logits).all() and np.isfinite(boxes).all(), name
            outs[name] = logits
    assert np.abs(outs['ReLU'] - g.gnn['logits']).max() < 2e-5
    for a in NAMES:
        if a not in ('ReLU', 'ReLU6'):    # this model's ReLU features stay below 6
            assert np.abs(outs[a] - outs['ReLU']).max() > 1e-3, a


def test_header_codes_equal_the_python_table():
    from pointgnn_b200 import _lib
    from pointgnn_b200.models import gnn
    with open(os.path.join(ROOT, 'include', 'pointgnn_b200.h')) as f:
        header = dict((k, int(v)) for k, v in re.findall(r'#define PG_ACT_(\w+) (\d+)\b', f.read()))
    names = {'NONE': 'NONE', 'RELU': 'ReLU', 'RELU6': 'ReLU6', 'LEAKY_RELU': 'LeakyReLU', 'ELU': 'ELU',
             'SIGMOID': 'Sigmoid', 'TANH': 'Tanh'}
    assert header['COUNT'] == len(names) == len(gnn.activation_fn_dict)
    for macro, name in names.items():
        assert gnn.activation_fn_dict[name] == header[macro] == getattr(_lib, 'PG_ACT_' + macro), name
    assert set(gnn.activation_fn_dict) == set(ACTIVATIONS)


def test_unknown_activation_name_is_a_key_error():
    from pointgnn_b200.models import gnn
    with pytest.raises(KeyError):
        gnn._check_types('NONE', 'Swish')
    with pytest.raises(NotImplementedError):
        gnn._check_types('BN', 'ReLU')
    assert gnn._check_types('NONE', 'Tanh') == gnn.activation_fn_dict['Tanh']

"""Every activation of the reference's table (gnn.py:24-32): ReLU, ReLU6, LeakyReLU, ELU, Sigmoid, Tanh and NONE.

The oracle (oracle/gnn.py) takes the activation from each ``*_activation_type`` of the config.  Its structure (concat
order, scopes, is_logits handling) is pinned by the ReLU goldens; the other activations are defined there from TF
1.15's documented behaviour (TF cannot run here and no shipped checkpoint was trained with them).  The GPU tests
compare the kernels against it."""
import copy
import os
import re

import numpy as np
import pytest

from oracle import gnn as ognn
from oracle.gnn import ACTIVATIONS, NAMES, activate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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
    logits, boxes = ognn.predict(g.weights, g.layer_configs, g.config['num_classes'], 7, g.graph['intensity'], coords,
                                 keypoints, edges)
    assert np.abs(logits - g.gnn['logits']).max() < 2e-5
    assert np.abs(boxes - g.gnn['boxes']).max() < 2e-5


def test_activation_oracle_runs_every_activation():
    """car_auto_T1 (one GNN iteration) with its own weights, every *_activation_type set to each entry in turn."""
    from conftest import load_golden
    g = load_golden('car_auto_T1_train')
    coords, keypoints, edges = g.graph_tuple()
    outs = {}
    for name in NAMES:
        lcs = with_activation(g.layer_configs, name)
        logits, boxes = ognn.predict(g.weights, lcs, g.config['num_classes'], 7, g.graph['intensity'], coords,
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

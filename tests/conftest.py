import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on the H100)')


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


class Golden(object):
    """One reference configuration: frozen config, trained weights, pinned graph + oracle outputs."""

    def __init__(self, name):
        self.name = name
        graph_name = name if name.startswith('ped') else 'car_auto_T3_train'   # car checkpoints share one graph
        with open(os.path.join(GOLDEN, 'config_%s.json' % name)) as f:
            self.config = json.load(f)
        self.weights = dict(np.load(os.path.join(GOLDEN, 'weights_%s.npz' % name)))
        self.graph = dict(np.load(os.path.join(GOLDEN, 'graph_%s.npz' % graph_name)))
        self.gnn = dict(np.load(os.path.join(GOLDEN, 'gnn_%s.npz' % name)))

    @property
    def layer_configs(self):
        return self.config['model_kwargs']['layer_configs']

    @property
    def graph_kwargs(self):
        return self.config['runtime_graph_gen_kwargs']

    def graph_tuple(self):
        """(vertex_coord_list, keypoint_indices_list, edges_list) in the reference's layout."""
        xyz = self.graph['xyz']
        kp = self.graph['keypoint_idx'].astype(np.int64)
        kxyz = xyz[kp]
        coords = [xyz, kxyz, kxyz]
        keypoints = [kp[:, None], np.arange(len(kp), dtype=np.int64)[:, None]]
        edges = [self.graph['edges0'].astype(np.int64), self.graph['edges1'].astype(np.int64)]
        return coords, keypoints, edges


_cache = {}


def load_golden(name):
    if name not in _cache:
        _cache[name] = Golden(name)
    return _cache[name]


ALL_CHECKPOINTS = ['car_auto_T0_train', 'car_auto_T1_train', 'car_auto_T2_train', 'car_auto_T3_train',
                   'car_auto_T3_trainval', 'car_fixed_T3_train', 'ped_cyl_auto_T3_trainval']


@pytest.fixture(scope='session')
def car():
    return load_golden('car_auto_T3_train')


@pytest.fixture(scope='session')
def ped():
    return load_golden('ped_cyl_auto_T3_trainval')

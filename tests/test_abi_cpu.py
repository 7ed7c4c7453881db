"""CPU tests of the drop-in boundary: the C-ABI library loads and exports every symbol the
header declares; the Python mirror keeps the reference's names; nothing falls back to the CPU."""
import inspect
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_text():
    with open(os.path.join(ROOT, 'include', 'pointgnn_b200.h')) as f:
        return f.read()


def _header_symbols():
    return sorted(set(re.findall(r'PG_API\s+[\w\s\*]+?\b(pg_\w+)\s*\(', _header_text())))


def test_library_exports_every_parsed_prototype():
    from pointgnn_b200 import _lib
    lib = _lib.load()
    syms = _header_symbols()
    assert len(syms) >= 12
    # one parsed prototype per PG_API declaration, and the library exports each with that prototype's arity
    assert len(re.findall(r'^PG_API\b', _header_text(), re.M)) == len(_lib.PROTOTYPES)
    assert sorted(_lib.PROTOTYPES) == syms
    for s in syms:
        assert hasattr(lib, s), 'libpointgnn_b200.so does not export %s' % s
        assert len(getattr(lib, s).argtypes) == len(_lib.PROTOTYPES[s][1])
    assert lib.pg_version() == 1
    assert lib.pg_last_error() == b''


def test_header_parser():
    """Integer #defines (negative, hex) become constants, macros do not; a type the binding does not know, or a
    declaration it cannot read, is an ImportError naming it - never an untyped pointer."""
    from pointgnn_b200 import _lib
    prototypes, constants = _lib.parse_header('''
        #define PG_API __attribute__((visibility("default")))
        #define PG_A (-4)   /* comment */
        #define PG_B 0x200
        #define PG_C 16
        #define PG_F(code) (PG_B | ((code) << PG_C))
        PG_API const char* pg_x(void);   /* PG_API int pg_in_comment(void); */
        PG_API int pg_y(const float* const* w_host, pg_layer **out, void* stream);''')
    assert constants == {'PG_A': -4, 'PG_B': 0x200, 'PG_C': 16}
    assert prototypes == {'pg_x': ('const char*', ()),
                          'pg_y': ('int', (('const float* const*', 'w_host'), ('pg_layer**', 'out'),
                                           ('void*', 'stream')))}
    for params in ((('const half*', 'x'),), (('void*', 'x'),), (('int64_t*', 'x'),), (('const uint8_t*', 'x_host'),)):
        with pytest.raises(ImportError, match=r'pg_z.*x'):
            _lib._bind('pg_z', 'int', params)
    with pytest.raises(ImportError, match='pg_q'):
        _lib.parse_header('PG_API int pg_q(int32_t);')


def test_call_binds_arguments_by_name(monkeypatch):
    """_call rejects a missing, an extra and a misspelt argument name before it converts anything or calls the
    library."""
    from pointgnn_b200 import _lib
    monkeypatch.setattr(_lib, 'load', lambda: pytest.fail('the library was called'))
    args = dict(src=object(), dst=object(), num_edges=0, num_src=0, num_dst=0)
    missing = {k: v for k, v in args.items() if k != 'num_dst'}
    misspelt = {('dest' if k == 'dst' else k): v for k, v in args.items()}
    for bad in (missing, dict(args, capacity=0), misspelt):
        with pytest.raises(TypeError, match='pg_check_edges'):
            _lib._call('pg_check_edges', **bad)


def test_no_cpu_fallback():
    from pointgnn_b200 import _lib
    x = torch.zeros(4, 3)
    with pytest.raises(TypeError):
        _lib.fully_connected(x, torch.zeros(3, 2), torch.zeros(2), True)
    import pointgnn_b200
    src = open(os.path.join(ROOT, 'point-gnn_b200', '_lib.py')).read()
    for mod in ('models/gnn.py', 'models/graph_gen.py', 'models/models.py', '_lib.py'):
        text = open(os.path.join(ROOT, 'point-gnn_b200', mod)).read()
        assert 'import oracle' not in text and 'from oracle' not in text, 'product path must not use the oracle'


def test_reference_api_surface():
    from pointgnn_b200.models import gnn, graph_gen, models
    # names and argument lists of the reference (gnn.py:222-232, :298-313, :133-135; graph_gen.py:155-157)
    sig = inspect.signature(gnn.PointSetPooling.apply_regular)
    assert list(sig.parameters)[1:5] == ['point_features', 'point_coordinates', 'keypoint_indices', 'set_indices']
    sig = inspect.signature(gnn.GraphNetAutoCenter.apply_regular)
    assert list(sig.parameters)[1:5] == ['input_vertex_features', 'input_vertex_coordinates', 'NOT_USED', 'edges']
    assert 'auto_offset_MLP_feature_activation_type' in sig.parameters
    sig = inspect.signature(gnn.ClassAwarePredictor.apply_regular)
    assert list(sig.parameters)[1:4] == ['features', 'num_classes', 'box_encoding_len']
    sig = inspect.signature(graph_gen.gen_multi_level_local_graph_v3)
    assert list(sig.parameters)[:5] == ['points_xyz', 'base_voxel_size', 'level_configs', 'add_rnd3d',
                                        'downsample_method']
    assert graph_gen.get_graph_generate_fn('multi_level_local_graph_v3') is graph_gen.gen_multi_level_local_graph_v3
    with pytest.raises(KeyError):
        graph_gen.get_graph_generate_fn('nope')
    with pytest.raises(KeyError):
        models.get_model('nope')
    m = models.get_model('multi_layer_fast_local_graph_model_v2')
    assert list(inspect.signature(m.predict).parameters)[1:6] == [
        't_initial_vertex_features', 't_vertex_coord_list', 't_keypoint_indices_list', 't_edges_list', 'is_training']


def test_variable_scope_names_follow_slim():
    from pointgnn_b200.models import gnn

    class FakeStore(object):
        def __init__(self):
            self.asked = []

        def get(self, name):
            self.asked.append(name)
            return name

    st = FakeStore()
    with gnn.variable_session(st):
        with gnn.variable_scope('layer2'):
            gnn._next_fully_connected()
            gnn._next_fully_connected()
            with gnn.variable_scope('extract_vertex_features'):
                gnn._next_fully_connected()
                gnn._next_fully_connected()
            with gnn.variable_scope('combined_features'):
                gnn._next_fully_connected()
    assert st.asked == [
        'layer2/fully_connected/weights', 'layer2/fully_connected/biases',
        'layer2/fully_connected_1/weights', 'layer2/fully_connected_1/biases',
        'layer2/extract_vertex_features/fully_connected/weights', 'layer2/extract_vertex_features/fully_connected/biases',
        'layer2/extract_vertex_features/fully_connected_1/weights',
        'layer2/extract_vertex_features/fully_connected_1/biases',
        'layer2/combined_features/fully_connected/weights', 'layer2/combined_features/fully_connected/biases']
    with pytest.raises(RuntimeError):
        gnn._next_fully_connected()


def test_checkpoint_variable_names_cover_config(car, ped):
    """Every variable the forward pass will ask for exists in the reference checkpoint."""
    from pointgnn_b200.models import gnn
    for g in (car, ped):
        names = set(g.weights)
        for lc in g.layer_configs[:-1]:
            s = lc['scope']
            if lc['type'] == 'scatter_max_point_set_pooling':
                n = len(lc['kwargs']['point_MLP_depth_list'])
                assert s + '/extract_vertex_features/fully_connected_%d/weights' % (n - 1) in names
            else:
                assert s + '/fully_connected_1/weights' in names          # auto-offset MLP
                assert g.weights[s + '/extract_vertex_features/fully_connected/weights'].shape[0] == \
                    g.weights[s + '/extract_vertex_features/fully_connected/weights'].shape[1] + 3
        assert 'output/predictor/loc/cls_%d/fully_connected_2/weights' % (g.config['num_classes'] - 1) in names


def test_training_only_paths_raise():
    from pointgnn_b200.models import graph_gen
    if torch.cuda.is_available():
        pytest.skip('argument checks below are reached before any device work only on CPU boxes')
    with pytest.raises((NotImplementedError, RuntimeError)):
        graph_gen.gen_multi_level_local_graph_v3(np.zeros((4, 3), np.float32), 0.8, [], downsample_method='random')


def test_prefetcher_has_no_cpu_path():
    """utils/prefetch.py overlaps GPU work with GPU work; without a CUDA device it must refuse, not fall back."""
    import torch
    if torch.cuda.is_available():
        pytest.skip('CUDA present')
    from pointgnn_b200.utils.prefetch import GraphPrefetcher
    with pytest.raises(RuntimeError):
        GraphPrefetcher(lambda *a, **k: None, {})

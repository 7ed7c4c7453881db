"""GNN layers and ops - same classes / functions / argument lists as the reference's
``models/gnn.py`` (/root/reference/models/gnn.py), executing on hand-written sm_90a kernels.

The reference builds a TF-1 graph whose variables are created by ``slim.fully_connected``
inside nested ``tf.variable_scope``s; here the same scoping is reproduced eagerly so that the
reference's checkpoints load by variable name: ``variable_scope(name)`` pushes a scope,
every fully-connected layer draws the next ``fully_connected[_i]`` name of its scope, and
weights are looked up in the active ``VariableStore`` (name -> CUDA tensor).

When a layer is built from the default plugins (``multi_layer_neural_network_fn`` +
``graph_scatter_max_fn``, i.e. every layer type models.py:49-74 registers) its gather /
concat / edge-MLP / segment-max chain runs as ONE fused kernel (``pg_edge_mlp_max``); any
other plugin combination runs the same chain op by op, still on the GPU.
"""
import contextlib
import threading
from functools import partial  # noqa: F401  (re-exported for config code written against the reference)

import torch

from .. import _lib
from .. import get_precision


# ---------------------------------------------------------------------------------------------
# variable scoping (stand-in for tf.variable_scope + slim's layer naming)
# ---------------------------------------------------------------------------------------------
class VariableStore(object):
    """name -> CUDA tensor, e.g. 'layer2/extract_vertex_features/fully_connected_1/weights'."""

    def __init__(self, variables=None, device=None):
        self.vars = {}
        self.prepared = {}      # (kind, first variable, depth, precision, activation) -> _lib.PreparedLayer
        if variables:
            self.load(variables, device)

    def load(self, variables, device=None):
        self.prepared.clear()
        device = device or torch.device('cuda', torch.cuda.current_device())
        for name, value in variables.items():
            if not (name.endswith('/weights') or name.endswith('/biases')):
                continue
            t = torch.as_tensor(value)
            if t.dtype != torch.float32:
                continue
            self.vars[name] = t.to(device).contiguous()

    def get(self, name):
        if name not in self.vars:
            raise KeyError('variable %r not found in the checkpoint' % name)   # TF: NotFoundError
        return self.vars[name]


class _Ctx(threading.local):
    def __init__(self):
        self.store = None
        self.scope = []
        self.counters = {}
        self.trusted_edges = False     # set by model.predict once an edge list has been range-checked


_ctx = _Ctx()


@contextlib.contextmanager
def variable_session(store):
    """One model build: binds the weight store and resets slim's per-scope layer counters."""
    prev = (_ctx.store, _ctx.scope, _ctx.counters)
    _ctx.store, _ctx.scope, _ctx.counters = store, [], {}
    try:
        yield store
    finally:
        _ctx.store, _ctx.scope, _ctx.counters = prev


@contextlib.contextmanager
def variable_scope(name):
    _ctx.scope.append(name)
    try:
        yield
    finally:
        _ctx.scope.pop()


def _next_fully_connected_named():
    if _ctx.store is None:
        raise RuntimeError('no VariableStore bound: call inside model.predict / variable_session')
    scope = '/'.join(_ctx.scope)
    i = _ctx.counters.get(scope, 0)
    _ctx.counters[scope] = i + 1
    base = (scope + '/' if scope else '') + ('fully_connected' if i == 0 else 'fully_connected_%d' % i)
    return base, _ctx.store.get(base + '/weights'), _ctx.store.get(base + '/biases')


def _next_fully_connected():
    return _next_fully_connected_named()[1:]


def _take_mlp(num_layers):
    """The next ``num_layers`` slim.fully_connected variables of the current scope -> (names, weights, biases)."""
    names, ws, bs = [], [], []
    for _ in range(num_layers):
        n, w, b = _next_fully_connected_named()
        names.append(n)
        ws.append(w)
        bs.append(b)
    return names, ws, bs


def _prepared(kind, names, weights, biases, dims, activation):
    """The prepared (weights packed once) layer for these variables and this activation, cached on the bound
    VariableStore - the stand-in for TF creating / restoring its variables once and only computing at sess.run."""
    store = _ctx.store
    key = (kind, names[0], len(names), get_precision(), activation)
    layer = store.prepared.get(key)
    if layer is None:
        layer = _lib.PreparedLayer(kind, weights, biases, dims, get_precision(), activation)
        store.prepared[key] = layer
    return layer


def _mlp_dims(ws, bs, widths):
    dims = [ws[0].shape[0]] + [w.shape[1] for w in ws]
    for i, (w, b) in enumerate(zip(ws, bs)):
        assert w.shape[0] == dims[i] and b.numel() == dims[i + 1], 'inconsistent layer shapes in the checkpoint'
    assert dims[1:] == [int(k) for k in widths], 'checkpoint layer widths %s != configured %s' % (dims[1:], list(widths))
    return dims


# the reference's tables (gnn.py:17-32).  Every activation runs in the fused kernels (the name -> PG_ACT_* code
# table of the whole package); of the normalizations only 'NONE' is built
normalization_fn_dict = {'fused_BN_center': 'fused_BN_center', 'BN': 'BN', 'BN_center': 'BN_center',
                         'IN': 'IN', 'NONE': None}
activation_fn_dict = {'ReLU': _lib.PG_ACT_RELU, 'ReLU6': _lib.PG_ACT_RELU6, 'LeakyReLU': _lib.PG_ACT_LEAKY_RELU,
                      'ELU': _lib.PG_ACT_ELU, 'NONE': _lib.PG_ACT_NONE, 'Sigmoid': _lib.PG_ACT_SIGMOID,
                      'Tanh': _lib.PG_ACT_TANH}


def _check_types(normalization_type, activation_type):
    """-> the PG_ACT_* code of activation_type; an unknown name raises KeyError, as the reference's lookup does."""
    if normalization_fn_dict[normalization_type] is not None:
        raise NotImplementedError('normalization %r: every shipped config uses "NONE" '
                                  '(SURVEY fact 3); batch/instance norm are not built' % normalization_type)
    return activation_fn_dict[activation_type]


def multi_layer_fc_fn(sv, mask=None, Ks=(64, 32, 64), num_classes=4, is_logits=False, num_layer=4,
                      normalization_type="fused_BN_center", activation_type='ReLU'):
    """gnn.py:34-84."""
    assert len(sv.shape) == 2
    assert len(Ks) == num_layer - 1
    act = _check_types(normalization_type, activation_type)
    names, ws, bs = _take_mlp(num_layer)
    layer = _prepared(_lib.PG_LAYER_MLP, names, ws, bs, _mlp_dims(ws, bs, list(Ks) + [num_classes]), act)
    features = layer.mlp(sv.contiguous(), last_linear=is_logits)
    if mask is not None:
        features = features * mask
    return features


def multi_layer_neural_network_fn(features, Ks=(64, 32, 64), is_logits=False,
                                  normalization_type="fused_BN_center", activation_type='ReLU',
                                  residual=None):
    """gnn.py:86-104.  ``residual`` (extension): added to the last layer's output in-kernel."""
    assert len(features.shape) == 2
    act = _check_types(normalization_type, activation_type)
    names, ws, bs = _take_mlp(len(Ks))
    layer = _prepared(_lib.PG_LAYER_MLP, names, ws, bs, _mlp_dims(ws, bs, Ks), act)
    return layer.mlp(features.contiguous(), last_linear=is_logits, residual=residual)


def _take_mlp_weights(num_layers):
    return _take_mlp(num_layers)[1:]


def graph_scatter_max_fn(point_features, point_centers, num_centers):
    """gnn.py:106-109 (tf.math.unsorted_segment_max; empty segment -> float lowest)."""
    centers = point_centers.reshape(-1).to(torch.int32).contiguous()
    return _lib.scatter_max(point_features.contiguous(), centers, int(num_centers))


def graph_scatter_sum_fn(point_features, point_centers, num_centers):
    """gnn.py:111-114 (tf.math.unsorted_segment_sum; empty segment -> 0).  No shipped config selects it; as an
    ``aggregation_fn`` plug-in it runs the layer op by op (the fused kernels implement the max)."""
    centers = point_centers.reshape(-1).to(torch.int32).contiguous()
    return _lib.scatter_sum(point_features.contiguous(), centers, int(num_centers))


def graph_scatter_mean_fn(point_features, point_centers, num_centers):
    """gnn.py:116-119 (tf.math.unsorted_segment_mean; empty segment -> 0)."""
    centers = point_centers.reshape(-1).to(torch.int32).contiguous()
    return _lib.scatter_sum(point_features.contiguous(), centers, int(num_centers), mean=True)


def _i32(t):
    return t.to(torch.int32).contiguous() if (t.dtype != torch.int32 or not t.is_contiguous()) else t


class ClassAwarePredictor(object):
    """gnn.py:121-163."""

    def __init__(self, cls_fn, loc_fn):
        self._cls_fn = cls_fn
        self._loc_fn = loc_fn

    def _head_width(self):
        """H when cls_fn / loc_fn are the registry's ``partial(multi_layer_fc_fn, Ks=(H,), num_layer=2)`` /
        ``partial(multi_layer_fc_fn, Ks=(H, H), num_layer=3)`` (models.py:60-64), else None."""
        c, l = self._cls_fn, self._loc_fn
        if not (isinstance(c, partial) and isinstance(l, partial) and c.func is multi_layer_fc_fn
                and l.func is multi_layer_fc_fn and not c.args and not l.args):
            return None
        ck, lk = c.keywords, l.keywords
        if set(ck) != {'Ks', 'num_layer'} or set(lk) != {'Ks', 'num_layer'}:
            return None
        if ck['num_layer'] != 2 or lk['num_layer'] != 3 or len(ck['Ks']) != 1 or len(lk['Ks']) != 2:
            return None
        h = int(ck['Ks'][0])
        return h if (int(lk['Ks'][0]) == h and int(lk['Ks'][1]) == h) else None

    def apply_regular(self, features, num_classes, box_encoding_len,
                      normalization_type='fused_BN_center', activation_type='ReLU'):
        h = self._head_width()
        if h is not None and normalization_type == 'NONE':
            act = _check_types(normalization_type, activation_type)
            # all heads in two launches per column group: the C + 1 first layers as ONE concatenated GEMM, then
            # one kernel for every remaining (tiny) layer, the softmax and the [K, C, box] stacking
            names, ws, bs = [], [], []
            with variable_scope('predictor'):
                with variable_scope('cls'):
                    n, w, b = _take_mlp(2)
                    names, ws, bs = names + n, ws + w, bs + b
                with variable_scope('loc'):
                    for class_idx in range(num_classes):
                        with variable_scope('cls_%d' % class_idx):
                            n, w, b = _take_mlp(3)
                            names, ws, bs = names + n, ws + w, bs + b
            d = ws[0].shape[0]
            assert tuple(ws[1].shape) == (h, num_classes) and tuple(ws[0].shape) == (d, h)
            for class_idx in range(num_classes):
                w0, w1, w2 = ws[2 + 3 * class_idx:5 + 3 * class_idx]
                assert tuple(w0.shape) == (d, h) and tuple(w1.shape) == (h, h) and tuple(w2.shape) == (h, box_encoding_len)
            layer = _prepared(_lib.PG_LAYER_PREDICTOR, names, ws, bs, [d, h, num_classes, box_encoding_len], act)
            logits, box_encodings, probs = layer.predictor(features.contiguous())
            logits._pg_probs = (probs, logits._version)      # models.postprocess returns these (softmax fused)
            return logits, box_encodings
        box_encodings_list = []
        with variable_scope('predictor'):
            with variable_scope('cls'):
                logits = self._cls_fn(features, num_classes=num_classes, is_logits=True,
                                      normalization_type=normalization_type,
                                      activation_type=activation_type)
            with variable_scope('loc'):
                for class_idx in range(num_classes):
                    with variable_scope('cls_%d' % class_idx):
                        box_encodings = self._loc_fn(features, num_classes=box_encoding_len, is_logits=True,
                                                     normalization_type=normalization_type,
                                                     activation_type=activation_type)
                        box_encodings_list.append(box_encodings.unsqueeze(1))
            box_encodings = torch.cat(box_encodings_list, dim=1)
        return logits, box_encodings


class PointSetPooling(object):
    """gnn.py:211-283."""

    def __init__(self, point_feature_fn=multi_layer_neural_network_fn,
                 aggregation_fn=graph_scatter_max_fn, output_fn=multi_layer_neural_network_fn):
        self._point_feature_fn = point_feature_fn
        self._aggregation_fn = aggregation_fn
        self._output_fn = output_fn

    def _fusable(self, normalization_type):
        return (self._point_feature_fn is multi_layer_neural_network_fn
                and self._aggregation_fn is graph_scatter_max_fn
                and normalization_type == 'NONE')

    def apply_regular(self, point_features, point_coordinates, keypoint_indices, set_indices,
                      point_MLP_depth_list=None, point_MLP_normalization_type='fused_BN_center',
                      point_MLP_activation_type='ReLU', output_MLP_depth_list=None,
                      output_MLP_normalization_type='fused_BN_center', output_MLP_activation_type='ReLU'):
        num_keypoints = keypoint_indices.shape[0]
        src, dst = set_indices[:, 0], set_indices[:, 1]
        with variable_scope('extract_vertex_features'):
            if self._fusable(point_MLP_normalization_type):
                act = _check_types(point_MLP_normalization_type, point_MLP_activation_type)
                names, ws, bs = _take_mlp(len(point_MLP_depth_list))
                dims = [point_features.shape[1] + 3] + [int(k) for k in point_MLP_depth_list]
                assert _mlp_dims(ws, bs, point_MLP_depth_list) == dims, 'point MLP input width mismatch'
                layer = _prepared(_lib.PG_LAYER_EDGE_POOL, names, ws, bs, dims, act)
                set_features = layer.edge_mlp_max(
                    point_features.contiguous(), point_coordinates.contiguous(), point_coordinates.contiguous(),
                    _i32(keypoint_indices.reshape(-1)), _i32(src), _i32(dst), num_keypoints,
                    trusted=_ctx.trusted_edges)
            else:
                # op-by-op composition, gnn.py:256-277
                psf = _lib.gather_rows(point_features.contiguous(), _i32(src))
                psc = _lib.gather_rows(point_coordinates.contiguous(), _i32(src))
                kidx = _i32(keypoint_indices.reshape(-1))[dst.long()]
                kc = _lib.gather_rows(point_coordinates.contiguous(), _i32(kidx))
                x = torch.cat([psf, psc - kc], dim=-1).contiguous()
                x = self._point_feature_fn(x, Ks=point_MLP_depth_list, is_logits=False,
                                           normalization_type=point_MLP_normalization_type,
                                           activation_type=point_MLP_activation_type)
                set_features = self._aggregation_fn(x, dst, num_keypoints)
        with variable_scope('combined_features'):
            set_features = self._output_fn(set_features, Ks=output_MLP_depth_list, is_logits=False,
                                           normalization_type=output_MLP_normalization_type,
                                           activation_type=output_MLP_activation_type)
        return set_features


class GraphNetAutoCenter(object):
    """gnn.py:285-373."""

    def __init__(self, edge_feature_fn=multi_layer_neural_network_fn, aggregation_fn=graph_scatter_max_fn,
                 update_fn=multi_layer_neural_network_fn, auto_offset_fn=multi_layer_neural_network_fn):
        self._edge_feature_fn = edge_feature_fn
        self._aggregation_fn = aggregation_fn
        self._update_fn = update_fn
        self._auto_offset_fn = auto_offset_fn

    def _fusable(self, normalization_type):
        return (self._edge_feature_fn is multi_layer_neural_network_fn
                and self._aggregation_fn is graph_scatter_max_fn
                and normalization_type == 'NONE')

    def apply_regular(self, input_vertex_features, input_vertex_coordinates, NOT_USED, edges,
                      edge_MLP_depth_list=None, edge_MLP_normalization_type='fused_BN_center',
                      edge_MLP_activation_type='ReLU', update_MLP_depth_list=None,
                      update_MLP_normalization_type='fused_BN_center', update_MLP_activation_type='ReLU',
                      auto_offset=False, auto_offset_MLP_depth_list=None,
                      auto_offset_MLP_normalization_type='fused_BN_center',
                      auto_offset_MLP_feature_activation_type='ReLU'):
        num_vertices = input_vertex_features.shape[0]
        src, dst = edges[:, 0], edges[:, 1]
        source_coordinates = input_vertex_coordinates.contiguous()          # gnn.py:339: un-offset
        dest_coordinates = source_coordinates
        if auto_offset:                                                     # gnn.py:341-346
            if self._auto_offset_fn is multi_layer_neural_network_fn:
                dest_coordinates = self._auto_offset_fn(
                    input_vertex_features, Ks=auto_offset_MLP_depth_list, is_logits=True,
                    normalization_type=auto_offset_MLP_normalization_type,
                    activation_type=auto_offset_MLP_feature_activation_type,
                    residual=source_coordinates)                            # coords + offset, fused
            else:
                offset = self._auto_offset_fn(
                    input_vertex_features, Ks=auto_offset_MLP_depth_list, is_logits=True,
                    normalization_type=auto_offset_MLP_normalization_type,
                    activation_type=auto_offset_MLP_feature_activation_type)
                dest_coordinates = (source_coordinates + offset).contiguous()
        with variable_scope('extract_vertex_features'):
            if self._fusable(edge_MLP_normalization_type):
                act = _check_types(edge_MLP_normalization_type, edge_MLP_activation_type)
                names, ws, bs = _take_mlp(len(edge_MLP_depth_list))
                dims = [input_vertex_features.shape[1] + 3] + [int(k) for k in edge_MLP_depth_list]
                assert _mlp_dims(ws, bs, edge_MLP_depth_list) == dims, 'edge MLP input width mismatch'
                layer = _prepared(_lib.PG_LAYER_EDGE_GNN, names, ws, bs, dims, act)
                aggregated_edge_features = layer.edge_mlp_max(
                    input_vertex_features.contiguous(), source_coordinates, dest_coordinates, None, _i32(src),
                    _i32(dst), num_vertices, trusted=_ctx.trusted_edges)
            else:
                # op-by-op composition, gnn.py:338-365
                s_feat = _lib.gather_rows(input_vertex_features.contiguous(), _i32(src))
                s_coord = _lib.gather_rows(source_coordinates, _i32(src))
                d_coord = _lib.gather_rows(dest_coordinates, _i32(dst))
                x = torch.cat([s_feat, s_coord - d_coord], dim=-1).contiguous()
                x = self._edge_feature_fn(x, Ks=edge_MLP_depth_list, is_logits=False,
                                          normalization_type=edge_MLP_normalization_type,
                                          activation_type=edge_MLP_activation_type)
                aggregated_edge_features = self._aggregation_fn(x, dst, num_vertices)
        with variable_scope('combined_features'):
            if self._update_fn is multi_layer_neural_network_fn:
                output_vertex_features = self._update_fn(
                    aggregated_edge_features, Ks=update_MLP_depth_list, is_logits=True,
                    normalization_type=update_MLP_normalization_type,
                    activation_type=update_MLP_activation_type,
                    residual=input_vertex_features.contiguous())            # gnn.py:372, fused
            else:
                update_features = self._update_fn(
                    aggregated_edge_features, Ks=update_MLP_depth_list, is_logits=True,
                    normalization_type=update_MLP_normalization_type,
                    activation_type=update_MLP_activation_type)
                output_vertex_features = update_features + input_vertex_features
        return output_vertex_features

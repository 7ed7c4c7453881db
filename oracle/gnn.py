"""CPU oracle for the GNN half of the hot path (reference models/gnn.py, models/models.py).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Line-by-line NumPy restatement, in
fp32 (dtype=np.float64 gives the "exact" arithmetic used to size tolerances), of

* multi_layer_neural_network_fn      gnn.py:86-104
* multi_layer_fc_fn                  gnn.py:34-84
* graph_scatter_{max,sum,mean}_fn    gnn.py:106-119  (tf.math.unsorted_segment_*:
                                     an empty segment -> numeric_limits<float>::lowest()
                                     for the max, 0 for the sum and the mean)
* ClassAwarePredictor.apply_regular  gnn.py:133-163
* ClassAwareSeparatedPredictor       gnn.py:177-209
* PointSetPooling.apply_regular      gnn.py:222-283
* GraphNetAutoCenter.apply_regular   gnn.py:298-373
* MultiLayerFastLocalGraphModelV2.predict / postprocess   models.py:79-168

``slim.fully_connected`` = act(x @ W + b) with W stored [in, out].  Every activation of
the reference's table (gnn.py:24-32) and every aggregation is an argument; the shipped
configs use normalization 'NONE', activation 'ReLU' and the max (SURVEY fact 3), the
combination the goldens pin.  The normalisers are not implemented.  Variable names follow
TF-slim scoping so the reference's checkpoints load unchanged:
'<scope>/fully_connected[_i]/{weights,biases}'.

``fp16=True`` is the library's FP16 arithmetic (precision code 2, ``set_precision('fp16')``).
It rounds exactly where the kernels round and nowhere else: every tensor-core operand (A and W)
is clipped to +-65504 and rounded once to ``np.float16``; products and sums are exact (float64)
and the accumulator is rounded once to fp32; bias, activation, residual and the aggregation follow
in fp32.  Which layers are tensor-core layers follows the library's routing (pg_tc.cu):
``fc_uses_tc`` for the dense layers, every layer after the first of a ReLU pooling MLP on one
feature channel (``pool_uses_tc``), the hoisted ``P = F @ W1[:C] + b1`` GEMM and the second layer
of a two-layer GNN edge MLP whose column groups of W keep resident in shared memory
(``gnn_uses_tc``), and the concatenated first layers of the class-aware predictor; the narrow
heads and the predictor's head kernel stay fp32.  Two places change structure with it: the GNN
edge layer is computed the way its kernel computes it, A = act(P[src] + (x_src - x_dst') @ W1[C:])
in fp32, rounded once; and the predictor's fused route runs every layer after a head's first in
fp32.  BF16x3 has no oracle of its own: it is held to the fp32 one.
"""
import numpy as np

NAMES = ['NONE', 'ReLU', 'ReLU6', 'LeakyReLU', 'ELU', 'Sigmoid', 'Tanh']
AGGREGATIONS = ('max', 'sum', 'mean')
F16_MAX = 65504.0
MAX_NT = 304                 # widest padded N of one tensor-core launch
SMEM_LIMIT = 227 * 1024      # shared memory a CTA may use


def _elu(x):
    with np.errstate(over='ignore'):
        return np.where(x > 0, x, np.exp(np.minimum(x, 0)) - x.dtype.type(1))


def _sigmoid(x):
    with np.errstate(over='ignore'):
        return x.dtype.type(1) / (x.dtype.type(1) + np.exp(-x))


# tf.nn.relu, relu6, leaky_relu(alpha=0.01) (gnn.py:28), elu (exp(x) - 1 below zero), sigmoid, tanh; None = linear.
# TF 1.15's documented behaviour: TF cannot run here and no shipped checkpoint was trained with the others.
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


# ---- FP16 rounding and the library's routing ----------------------------------------------------------------------
def f16(a):
    """A tensor-core operand: clipped to FP16's range, rounded once to nearest, as float64."""
    a = np.clip(np.asarray(a, dtype=np.float32), -F16_MAX, F16_MAX)
    return a.astype(np.float16).astype(np.float64)


def tc_gemm(x, w):
    """One FP16 tensor-core GEMM: FP16 operands, exact products and sums, one rounding to fp32."""
    return (f16(x) @ f16(w)).astype(np.float32)


def fc_uses_tc(k, n):
    """pg_tc.cu fc_uses_tc: narrow / shallow layers stay on the fp32 FFMA kernel."""
    return k % 4 == 0 and n >= 8 and (k + 15) // 16 * 16 >= 64


def _column_blocks(n, max_w):
    nb = -(-n // max_w)
    w = (-(-n // nb) + 15) // 16 * 16
    return [(c, min(n, c + w)) for c in range(0, n, w)]


def _ni(n):
    npad = (n + 15) // 16 * 16
    return 64 if npad <= 64 else 128 if npad <= 128 else 96 if npad <= 192 else 128 if npad <= 256 else 152


def gnn_w_resident(kp, n, max_w):
    """Every column group of the FP16 W image (kp x ni x 2 B) fits shared memory with the gather stages."""
    return all((kp // 16) * _ni(c1 - c0) * 32 + 3 * 4096 + 8 <= SMEM_LIMIT for c0, c1 in _column_blocks(n, max_w))


def pool_uses_tc(dims, act):
    """prepare_edge's pooling route: the on-chip chain is built for ReLU on one feature channel."""
    L = len(dims) - 1
    if L < 2 or act != 'ReLU' or dims[0] != 4:
        return False
    for l in range(1, L):
        if l > 1 and dims[l] % 4:
            return False
        if l + 1 < L and (dims[l + 1] > MAX_NT or dims[l + 1] % 4):
            return False
    return True


def gnn_uses_tc(dims):
    """prepare_edge's GNN route: two layers, W2's column groups resident (152- or 64-wide)."""
    if len(dims) != 3:
        return False
    kp = (dims[1] + 15) // 16 * 16
    return gnn_w_resident(kp, dims[2], MAX_NT) or gnn_w_resident(kp, dims[2], 64)


def _predictor_fused(d, h, c, box):
    """prepare_predictor: the concatenated first layers + the fp32 head kernel (H = 64, weights in shared memory)."""
    pad4 = lambda v: (v + 3) & ~3  # noqa: E731
    wfloats = pad4(h * c) + pad4(c) + c * (pad4(h * h) + pad4(h) + pad4(h * box) + pad4(box))
    smem = (pad4(wfloats) + 2 * 64 * 65 + 64 * 16) * 4
    return h == 64 and smem <= SMEM_LIMIT and fc_uses_tc(d, h)


# ---- dense layers -------------------------------------------------------------------------------------------------
class _Scope(object):
    """Mimics slim's per-variable_scope 'fully_connected', 'fully_connected_1', ... naming.  fp16: the arithmetic of
    the dense layers drawn from it, so the MLP functions keep the reference's signatures."""

    def __init__(self, weights, prefix, fp16=False):
        self.weights = weights
        self.prefix = prefix
        self.fp16 = fp16
        self.count = 0

    def sub(self, name):
        return _Scope(self.weights, self.prefix + '/' + name if self.prefix else name, self.fp16)

    def next_fc(self):
        name = 'fully_connected' if self.count == 0 else 'fully_connected_%d' % self.count
        self.count += 1
        base = self.prefix + '/' + name
        return self.weights[base + '/weights'], self.weights[base + '/biases']

    def take(self, n):
        """The next n layers' weights and biases as two lists."""
        ws, bs = zip(*[self.next_fc() for _ in range(n)])
        return list(ws), list(bs)


def _dense(x, w, b, act, tc=False):
    """act(x @ W + b) in x's dtype; tc: an FP16 tensor-core layer."""
    y = tc_gemm(x, w) if tc else x @ w.astype(x.dtype)
    return activate(act, y + b.astype(x.dtype)[None, :])


def dense(x, w, b, act, fp16=False):
    """One dense layer, routed as the library's dense kernel routes it."""
    return _dense(x, w, b, act, fp16 and fc_uses_tc(*w.shape))


def _fc(x, scope, act):
    w, b = scope.next_fc()
    assert x.shape[1] == w.shape[0], (x.shape, w.shape, scope.prefix)
    return dense(x, w, b, act, scope.fp16)


def _check_types(normalization_type, activation_type):
    assert normalization_type == 'NONE', 'only normalization NONE is used by the shipped configs'
    assert activation_type in ACTIVATIONS, activation_type


def multi_layer_neural_network_fn(features, scope, Ks=(64, 32, 64), is_logits=False,
                                  normalization_type='NONE', activation_type='ReLU'):
    """gnn.py:86-104."""
    assert len(features.shape) == 2
    _check_types(normalization_type, activation_type)
    for i in range(len(Ks)):
        last = i == len(Ks) - 1
        features = _fc(features, scope, 'NONE' if (is_logits and last) else activation_type)
        assert features.shape[1] == Ks[i]
    return features


def multi_layer_fc_fn(sv, scope, Ks=(64, 32, 64), num_classes=4, is_logits=False, num_layer=4,
                      normalization_type='NONE', activation_type='ReLU'):
    """gnn.py:34-84 (mask unused by the predictor)."""
    assert len(sv.shape) == 2
    assert len(Ks) == num_layer - 1
    _check_types(normalization_type, activation_type)
    features = sv
    for i in range(num_layer - 1):
        features = _fc(features, scope, activation_type)
    features = _fc(features, scope, 'NONE' if is_logits else activation_type)
    assert features.shape[1] == num_classes
    return features


# ---- aggregations -------------------------------------------------------------------------------------------------
def graph_scatter_max_fn(point_features, point_centers, num_centers):
    """gnn.py:106-109; tf.math.unsorted_segment_max semantics."""
    point_centers = np.asarray(point_centers).reshape(-1).astype(np.int64)
    lowest = np.finfo(point_features.dtype).min
    out = np.full((int(num_centers), point_features.shape[1]), lowest, dtype=point_features.dtype)
    if point_features.shape[0] == 0:
        return out
    if np.any(np.diff(point_centers) < 0):
        order = np.argsort(point_centers, kind='stable')
        point_centers = point_centers[order]
        point_features = point_features[order]
    starts = np.flatnonzero(np.concatenate([[True], point_centers[1:] != point_centers[:-1]]))
    out[point_centers[starts]] = np.maximum.reduceat(point_features, starts, axis=0)
    return out


def segment_reduce(x, dst, num, aggregation):
    """tf.math.unsorted_segment_max / _sum / _mean in x's dtype, dst in any order; an empty segment gives the lowest
    float (max) or 0 (sum, mean)."""
    dst = np.asarray(dst).reshape(-1).astype(np.int64)
    if aggregation == 'max':
        return graph_scatter_max_fn(x, dst, num)
    out = np.zeros((int(num), x.shape[1]), x.dtype)
    if len(dst):
        order = np.argsort(dst, kind='stable')
        d, xs = dst[order], x[order]
        starts = np.flatnonzero(np.concatenate([[True], d[1:] != d[:-1]]))
        out[d[starts]] = np.add.reduceat(xs, starts, axis=0)
    if aggregation == 'mean':
        out /= np.maximum(np.bincount(dst, minlength=int(num)), 1).astype(x.dtype)[:, None]
    return out


class _Reduction(object):
    """A segment reduction fed chunk by chunk: partial maxima or sums, the mean's division at the end."""

    def __init__(self, num, n, dtype, aggregation):
        assert aggregation in AGGREGATIONS, aggregation
        self.aggregation = aggregation
        self.count = np.zeros(int(num), np.int64)
        self.out = segment_reduce(np.zeros((0, n), dtype), [], num, 'max' if aggregation == 'max' else 'sum')

    def add(self, x, dst):
        part = segment_reduce(x, dst, self.out.shape[0], 'max' if self.aggregation == 'max' else 'sum')
        if self.aggregation == 'max':
            np.maximum(self.out, part, out=self.out)
        else:
            self.out += part
        self.count += np.bincount(np.asarray(dst, np.int64), minlength=self.out.shape[0])

    def result(self):
        if self.aggregation == 'mean':
            self.out /= np.maximum(self.count, 1).astype(self.out.dtype)[:, None]
        return self.out


def _chunks(n, chunk, fp16):
    """Edge chunks (bound the oracle's memory).  A sum depends on them: 2^16 edges, 2^15 under FP16."""
    chunk = chunk or (1 << 15 if fp16 else 1 << 16)
    for s in range(0, n, chunk):
        yield s, min(n, s + chunk)


# ---- edge layers, over weight lists -------------------------------------------------------------------------------
def pool_edge_layer(feat, xyz, kxyz, src, dst, num_dst, ws, bs, act='ReLU', aggregation='max', fp16=False,
                    chunk=None):
    """PointSetPooling's edge MLP and aggregation (gnn.py:256-277), pg_edge_mlp_max PG_EDGE_POOL: kxyz[dst] is a
    destination's keypoint coordinates."""
    dims = [ws[0].shape[0]] + [w.shape[1] for w in ws]
    tc = fp16 and pool_uses_tc(dims, act)
    red = _Reduction(num_dst, dims[-1], feat.dtype, aggregation)
    for s, e in _chunks(len(src), chunk, fp16):
        si, di = src[s:e], dst[s:e]
        x = np.concatenate([feat[si], xyz[si] - kxyz[di]], axis=-1)          # :256-267
        for l, (w, b) in enumerate(zip(ws, bs)):
            x = _dense(x, w, b, act, tc and l > 0)
        red.add(x, di)                                                       # :275-277
    return red.result()


def gnn_edge_layer(feat, xyz_src, xyz_dst, src, dst, num_dst, ws, bs, act='ReLU', aggregation='max', fp16=False,
                   chunk=None):
    """GraphNetAutoCenter's edge MLP and aggregation (gnn.py:338-365), pg_edge_mlp_max PG_EDGE_GNN: xyz_dst holds
    the offset coordinates."""
    dims = [ws[0].shape[0]] + [w.shape[1] for w in ws]
    c = feat.shape[1]
    tc = fp16 and gnn_uses_tc(dims)
    if tc:
        # the hoisted per-vertex table, itself a dense layer (linear)
        p = dense(feat, ws[0][:c], bs[0], 'NONE', fp16=True)
    red = _Reduction(num_dst, dims[-1], feat.dtype, aggregation)
    for s, e in _chunks(len(src), chunk, fp16):
        si, di = src[s:e], dst[s:e]
        d = xyz_src[si] - xyz_dst[di]                                        # :338-348 (un-offset - offset)
        if tc:
            x = activate(act, p[si] + d @ ws[0][c:].astype(np.float32))
            x = _dense(x, ws[1], bs[1], act, True)
        else:
            x = np.concatenate([feat[si], d], axis=-1)                       # :350-352
            for w, b in zip(ws, bs):
                x = _dense(x, w, b, act)
        red.add(x, di)                                                       # :362-365
    return red.result()


# ---- layers -------------------------------------------------------------------------------------------------------
def point_set_pooling(weights, scope_name, point_features, point_coordinates, keypoint_indices,
                      set_indices, point_MLP_depth_list=None, point_MLP_normalization_type='NONE',
                      point_MLP_activation_type='ReLU', output_MLP_depth_list=None,
                      output_MLP_normalization_type='NONE', output_MLP_activation_type='ReLU',
                      aggregation='max', fp16=False, chunk=None):
    """PointSetPooling.apply_regular, gnn.py:222-283."""
    _check_types(point_MLP_normalization_type, point_MLP_activation_type)
    set_indices = np.asarray(set_indices).astype(np.int64)
    kidx = np.asarray(keypoint_indices).astype(np.int64)[:, 0]
    ws, bs = _Scope(weights, scope_name).sub('extract_vertex_features').take(len(point_MLP_depth_list))
    set_features = pool_edge_layer(point_features, point_coordinates, point_coordinates[kidx], set_indices[:, 0],
                                   set_indices[:, 1], len(kidx), ws, bs, act=point_MLP_activation_type,
                                   aggregation=aggregation, fp16=fp16, chunk=chunk)
    sc = _Scope(weights, scope_name, fp16).sub('combined_features')
    return multi_layer_neural_network_fn(set_features, sc, Ks=output_MLP_depth_list,
                                         is_logits=False,
                                         normalization_type=output_MLP_normalization_type,
                                         activation_type=output_MLP_activation_type)


def graph_net_auto_center(weights, scope_name, input_vertex_features, input_vertex_coordinates,
                          NOT_USED, edges, edge_MLP_depth_list=None,
                          edge_MLP_normalization_type='NONE', edge_MLP_activation_type='ReLU',
                          update_MLP_depth_list=None, update_MLP_normalization_type='NONE',
                          update_MLP_activation_type='ReLU', auto_offset=False,
                          auto_offset_MLP_depth_list=None,
                          auto_offset_MLP_normalization_type='NONE',
                          auto_offset_MLP_feature_activation_type='ReLU', aggregation='max', fp16=False,
                          chunk=None):
    """GraphNetAutoCenter.apply_regular, gnn.py:298-373."""
    _check_types(edge_MLP_normalization_type, edge_MLP_activation_type)
    edges = np.asarray(edges).astype(np.int64)
    top = _Scope(weights, scope_name, fp16)
    coords = input_vertex_coordinates
    if auto_offset:                                                      # :341-346
        offset = multi_layer_neural_network_fn(
            input_vertex_features, top, Ks=auto_offset_MLP_depth_list, is_logits=True,
            normalization_type=auto_offset_MLP_normalization_type,
            activation_type=auto_offset_MLP_feature_activation_type)
        coords = input_vertex_coordinates + offset
    ws, bs = _Scope(weights, scope_name).sub('extract_vertex_features').take(len(edge_MLP_depth_list))
    agg = gnn_edge_layer(input_vertex_features, input_vertex_coordinates, coords, edges[:, 0], edges[:, 1],
                         input_vertex_features.shape[0], ws, bs, act=edge_MLP_activation_type,
                         aggregation=aggregation, fp16=fp16, chunk=chunk)
    sc = _Scope(weights, scope_name, fp16).sub('combined_features')
    update = multi_layer_neural_network_fn(agg, sc, Ks=update_MLP_depth_list, is_logits=True,
                                           normalization_type=update_MLP_normalization_type,
                                           activation_type=update_MLP_activation_type)
    return update + input_vertex_features                                # :372


def class_aware_predictor(weights, scope_name, features, num_classes, box_encoding_len,
                          normalization_type='NONE', activation_type='ReLU',
                          cls_Ks=(64,), loc_Ks=(64, 64), separated=False, fp16=False):
    """ClassAwarePredictor.apply_regular, gnn.py:133-163, or with separated=True
    ClassAwareSeparatedPredictor.apply_regular, gnn.py:177-209 (class c's loc head reads the c-th of C equal
    np.split slices), with the fns of models.py:60-74.  The library runs the separated predictor under FP16 as the
    shared one on zero-padded loc weights, so that is where the FP16 oracle computes it too."""
    assert not (separated and fp16), 'FP16: the shared predictor on zero-padded loc weights'
    pred = _Scope(weights, scope_name, fp16).sub('predictor')
    # FP16, prepare_predictor's fused route: a head's first layer is one of the concatenated tensor-core first
    # layers, its other layers run on the fp32 head kernel
    fused = fp16 and _predictor_fused(features.shape[1], cls_Ks[0], num_classes, box_encoding_len)

    def head(x, scope, Ks, n):
        kw = dict(num_classes=n, is_logits=True, normalization_type=normalization_type,
                  activation_type=activation_type)
        if fused:
            x = _fc(x, scope, activation_type)
            scope.fp16 = False
            return multi_layer_fc_fn(x, scope, Ks=Ks[1:], num_layer=len(Ks), **kw)
        return multi_layer_fc_fn(x, scope, Ks=Ks, num_layer=len(Ks) + 1, **kw)

    logits = head(features, pred.sub('cls'), cls_Ks, num_classes)
    loc_inputs = np.split(features, num_classes, axis=-1) if separated else [features] * num_classes
    boxes = [head(loc_inputs[c], pred.sub('loc').sub('cls_%d' % c), loc_Ks, box_encoding_len)[:, None, :]
             for c in range(num_classes)]
    return logits, np.concatenate(boxes, axis=1)


_PREDICTOR_KS = {
    'classaware_predictor': ((64,), (64, 64)),
    'classaware_predictor_128': ((128,), (128, 128)),
    'classaware_separated_predictor': ((64,), (64, 64)),
}


def predict(weights, layer_configs, num_classes, box_encoding_len, t_initial_vertex_features,
            t_vertex_coord_list, t_keypoint_indices_list, t_edges_list, dtype=np.float32,
            return_features=False, **options):
    """MultiLayerFastLocalGraphModelV2.predict, models.py:79-163.  options (aggregation, fp16, chunk) go to every
    point_set_pooling and graph_net_auto_center call, fp16 to the predictor as well.  Only the options given are
    passed, so without them a layer call carries the config's keywords alone, as in the reference."""
    fp16 = options.get('fp16', False)
    assert not fp16 or dtype == np.float32
    feats = np.asarray(t_initial_vertex_features, dtype=dtype)
    coords = [np.asarray(c, dtype=dtype) for c in t_vertex_coord_list]
    feature_list = [feats]
    for layer_config in layer_configs[:-1]:
        lvl = layer_config['graph_level']
        kw = dict(layer_config['kwargs'], **options)
        if layer_config['type'] == 'scatter_max_point_set_pooling':
            feats = point_set_pooling(weights, layer_config['scope'], feats, coords[lvl],
                                      t_keypoint_indices_list[lvl], t_edges_list[lvl], **kw)
        elif layer_config['type'] == 'scatter_max_graph_auto_center_net':
            feats = graph_net_auto_center(weights, layer_config['scope'], feats, coords[lvl],
                                          t_keypoint_indices_list[lvl], t_edges_list[lvl], **kw)
        else:
            raise KeyError(layer_config['type'])
        feature_list.append(feats)
    pc = layer_configs[-1]
    cls_Ks, loc_Ks = _PREDICTOR_KS[pc['type']]
    logits, boxes = class_aware_predictor(weights, pc['scope'], feats, num_classes,
                                          box_encoding_len, cls_Ks=cls_Ks, loc_Ks=loc_Ks,
                                          separated=pc['type'] == 'classaware_separated_predictor',
                                          fp16=fp16, **pc['kwargs'])
    if return_features:
        return logits, boxes, feature_list
    return logits, boxes


def postprocess(logits):
    """models.py:165-168: softmax over classes."""
    z = logits - logits.max(axis=-1, keepdims=True)
    e = np.exp(z)
    return e / e.sum(axis=-1, keepdims=True)

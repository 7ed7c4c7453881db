"""CPU oracle of the FP16 tensor-core arithmetic (precision code 2, ``set_precision('fp16')``).

Rounds exactly where the kernels round and nowhere else: every tensor-core operand (A and W) is clipped to
+-65504 and rounded once to ``np.float16``; products and sums are exact (float64) and the accumulator is rounded once
to fp32; bias, activation, residual and segment max follow in fp32.  Which layers are tensor-core layers follows the
library's own routing (pg_tc.cu): ``fc_uses_tc`` for the dense layers, every layer after the first of a ReLU pooling
MLP on one feature channel, the hoisted ``P = F @ W1[:C] + b1`` GEMM and the second layer of a two-layer GNN edge MLP
whose column groups of W keep resident in shared memory, and the concatenated first layers of the class-aware
predictor; the narrow heads and the predictor's head kernel stay fp32.  The GNN edge layer is computed the way its
kernel computes it: A = act(P[src] + (x_src - x_dst') @ W1[C:]) in fp32, rounded once.

The fp32 oracle (oracle/gnn.py) stays the reference for the fp32 and BF16x3 arithmetics; this module reuses its
slim scoping, its segment max and its predictor table.  Activations: test_activations_cpu's table."""
import numpy as np

from oracle import gnn as ognn
from test_activations_cpu import activate

F16_MAX = 65504.0
MAX_NT = 304                 # widest padded N of one tensor-core launch
SMEM_LIMIT = 227 * 1024      # shared memory a CTA may use
LOWEST = np.finfo(np.float32).min


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


def fc(x, w, b, act, residual=None):
    """act(x @ W + b) (+ residual) of one dense layer under precision 2."""
    x = np.asarray(x, dtype=np.float32)
    k, n = w.shape
    if fc_uses_tc(k, n):
        y = tc_gemm(x, w) + b.astype(np.float32)[None, :]
    else:
        y = x @ w.astype(np.float32) + b.astype(np.float32)[None, :]
    y = activate(act, y)
    return y if residual is None else y + residual


def mlp(x, scope, Ks, is_logits, act, residual=None):
    """multi_layer_neural_network_fn / multi_layer_fc_fn (gnn.py:34-104) on the dense layers."""
    for i in range(len(Ks)):
        last = i == len(Ks) - 1
        w, b = scope.next_fc()
        x = fc(x, w, b, 'NONE' if (is_logits and last) else act, residual if last else None)
        assert x.shape[1] == Ks[i]
    return x


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


def _chunks(n, chunk):
    for s in range(0, n, chunk):
        yield s, min(n, s + chunk)


def pool_edge_max(feat, xyz, kxyz, src, dst, num_dst, ws, bs, act='ReLU', chunk=1 << 15):
    """pg_edge_mlp_max PG_EDGE_POOL under precision 2: kxyz is the keypoints' coordinates (xyz_dst[kp[dst]])."""
    dims = [ws[0].shape[0]] + [w.shape[1] for w in ws]
    tc = pool_uses_tc(dims, act)
    out = np.full((int(num_dst), dims[-1]), LOWEST, np.float32)
    for s, e in _chunks(len(src), chunk):
        si, di = src[s:e], dst[s:e]
        x = np.concatenate([feat[si], xyz[si] - kxyz[di]], axis=1).astype(np.float32)
        for l, (w, b) in enumerate(zip(ws, bs)):
            if tc and l > 0:
                x = activate(act, tc_gemm(x, w) + b.astype(np.float32)[None, :])
            else:
                x = activate(act, x @ w.astype(np.float32) + b.astype(np.float32)[None, :])
        np.maximum(out, ognn.graph_scatter_max_fn(x, di, num_dst), out=out)
    return out


def gnn_edge_max(feat, xyz_src, xyz_dst, src, dst, num_dst, ws, bs, act='ReLU', chunk=1 << 15):
    """pg_edge_mlp_max PG_EDGE_GNN under precision 2 (xyz_dst: the offset coordinates)."""
    dims = [ws[0].shape[0]] + [w.shape[1] for w in ws]
    c = feat.shape[1]
    out = np.full((int(num_dst), dims[-1]), LOWEST, np.float32)
    tc = gnn_uses_tc(dims)
    if tc:
        # the hoisted per-vertex table, itself a dense layer (linear)
        p = fc(feat, ws[0][:c], bs[0], 'NONE')
    for s, e in _chunks(len(src), chunk):
        si, di = src[s:e], dst[s:e]
        d = (xyz_src[si] - xyz_dst[di]).astype(np.float32)
        if tc:
            x = activate(act, p[si] + d @ ws[0][c:].astype(np.float32))
            x = activate(act, tc_gemm(x, ws[1]) + bs[1].astype(np.float32)[None, :])
        else:
            x = np.concatenate([feat[si], d], axis=1).astype(np.float32)
            for w, b in zip(ws, bs):
                x = activate(act, x @ w.astype(np.float32) + b.astype(np.float32)[None, :])
        np.maximum(out, ognn.graph_scatter_max_fn(x, di, num_dst), out=out)
    return out


def _take(scope, n):
    ws, bs = [], []
    for _ in range(n):
        w, b = scope.next_fc()
        ws.append(w)
        bs.append(b)
    return ws, bs


def point_set_pooling(weights, scope_name, point_features, point_coordinates, keypoint_indices, set_indices,
                      point_MLP_depth_list=None, point_MLP_normalization_type='NONE', point_MLP_activation_type='ReLU',
                      output_MLP_depth_list=None, output_MLP_normalization_type='NONE',
                      output_MLP_activation_type='ReLU'):
    """PointSetPooling.apply_regular (gnn.py:222-283) under precision 2."""
    set_indices = np.asarray(set_indices).astype(np.int64)
    kidx = np.asarray(keypoint_indices).astype(np.int64)[:, 0]
    ws, bs = _take(ognn._Scope(weights, scope_name).sub('extract_vertex_features'), len(point_MLP_depth_list))
    set_features = pool_edge_max(point_features, point_coordinates, point_coordinates[kidx], set_indices[:, 0],
                                 set_indices[:, 1], len(kidx), ws, bs, point_MLP_activation_type)
    sc = ognn._Scope(weights, scope_name).sub('combined_features')
    return mlp(set_features, sc, output_MLP_depth_list, False, output_MLP_activation_type)


def graph_net_auto_center(weights, scope_name, input_vertex_features, input_vertex_coordinates, NOT_USED, edges,
                          edge_MLP_depth_list=None, edge_MLP_normalization_type='NONE', edge_MLP_activation_type='ReLU',
                          update_MLP_depth_list=None, update_MLP_normalization_type='NONE',
                          update_MLP_activation_type='ReLU', auto_offset=False, auto_offset_MLP_depth_list=None,
                          auto_offset_MLP_normalization_type='NONE', auto_offset_MLP_feature_activation_type='ReLU'):
    """GraphNetAutoCenter.apply_regular (gnn.py:298-373) under precision 2."""
    edges = np.asarray(edges).astype(np.int64)
    top = ognn._Scope(weights, scope_name)
    coords = input_vertex_coordinates
    if auto_offset:
        coords = mlp(input_vertex_features, top, auto_offset_MLP_depth_list, True,
                     auto_offset_MLP_feature_activation_type, residual=input_vertex_coordinates)
    ws, bs = _take(ognn._Scope(weights, scope_name).sub('extract_vertex_features'), len(edge_MLP_depth_list))
    agg = gnn_edge_max(input_vertex_features, input_vertex_coordinates, coords, edges[:, 0], edges[:, 1],
                       input_vertex_features.shape[0], ws, bs, edge_MLP_activation_type)
    sc = ognn._Scope(weights, scope_name).sub('combined_features')
    return mlp(agg, sc, update_MLP_depth_list, True, update_MLP_activation_type, residual=input_vertex_features)


def _predictor_fused(d, h, c, box):
    """prepare_predictor: the concatenated first layers + the fp32 head kernel (H = 64, weights in shared memory)."""
    pad4 = lambda v: (v + 3) & ~3  # noqa: E731
    wfloats = pad4(h * c) + pad4(c) + c * (pad4(h * h) + pad4(h) + pad4(h * box) + pad4(box))
    smem = (pad4(wfloats) + 2 * 64 * 65 + 64 * 16) * 4
    return h == 64 and smem <= SMEM_LIMIT and fc_uses_tc(d, h)


def class_aware_predictor(weights, scope_name, features, num_classes, box_encoding_len, normalization_type='NONE',
                          activation_type='ReLU', cls_Ks=(64,), loc_Ks=(64, 64)):
    """ClassAwarePredictor.apply_regular (gnn.py:133-163) under precision 2."""
    pred = ognn._Scope(weights, scope_name).sub('predictor')
    h, act = cls_Ks[0], activation_type
    fused = _predictor_fused(features.shape[1], h, num_classes, box_encoding_len)

    def head(scope, n_layers):
        ws, bs = _take(scope, n_layers)
        x = fc(features, ws[0], bs[0], act)            # a first layer: a tensor-core layer in both routes here
        for i in range(1, n_layers):
            last = i == n_layers - 1
            a = 'NONE' if last else act
            if fused:                                  # predictor_heads_kernel: fp32
                x = activate(a, x @ ws[i].astype(np.float32) + bs[i].astype(np.float32)[None, :])
            else:
                x = fc(x, ws[i], bs[i], a)
        return x

    logits = head(pred.sub('cls'), len(cls_Ks) + 1)
    boxes = [head(pred.sub('loc').sub('cls_%d' % ci), len(loc_Ks) + 1)[:, None, :] for ci in range(num_classes)]
    return logits, np.concatenate(boxes, axis=1)


def predict(weights, layer_configs, num_classes, box_encoding_len, t_initial_vertex_features, t_vertex_coord_list,
            t_keypoint_indices_list, t_edges_list):
    """MultiLayerFastLocalGraphModelV2.predict (models.py:79-163) under precision 2."""
    feats = np.asarray(t_initial_vertex_features, dtype=np.float32)
    coords = [np.asarray(c, dtype=np.float32) for c in t_vertex_coord_list]
    for lc in layer_configs[:-1]:
        lvl, kw = lc['graph_level'], lc['kwargs']
        if lc['type'] == 'scatter_max_point_set_pooling':
            feats = point_set_pooling(weights, lc['scope'], feats, coords[lvl], t_keypoint_indices_list[lvl],
                                      t_edges_list[lvl], **kw)
        elif lc['type'] == 'scatter_max_graph_auto_center_net':
            feats = graph_net_auto_center(weights, lc['scope'], feats, coords[lvl], t_keypoint_indices_list[lvl],
                                          t_edges_list[lvl], **kw)
        else:
            raise KeyError(lc['type'])
    pc = layer_configs[-1]
    cls_Ks, loc_Ks = ognn._PREDICTOR_KS[pc['type']]
    return class_aware_predictor(weights, pc['scope'], feats, num_classes, box_encoding_len, cls_Ks=cls_Ks,
                                 loc_Ks=loc_Ks, **pc['kwargs'])

"""Model assembly - mirror of the forward half of the reference's ``models/models.py``
(/root/reference/models/models.py:23-168, 313-319): ``get_model(name)`` ->
``MultiLayerFastLocalGraphModelV2`` with ``predict`` / ``postprocess``.  The training loss
(models.py:170-311) is out of scope (SURVEY section 2).

Differences forced by running eagerly instead of building a TF-1 graph: weights are loaded
explicitly (``load_checkpoint`` / ``load_weights``) instead of through ``tf.train.Saver``, and
``predict`` takes arrays / tensors instead of placeholders.  NumPy inputs are copied to the GPU
and results returned as NumPy (the ``sess.run`` convention of run.py:252-260); CUDA tensors
stay on the device.
"""
from functools import partial

import numpy as np
import torch

from . import gnn
from .. import _lib
from ..utils import tf_checkpoint


class MultiLayerFastLocalGraphModelV2(object):
    """models.py:23-168."""

    def __init__(self, num_classes, box_encoding_len, regularizer_type=None,
                 regularizer_kwargs=None, layer_configs=None, mode=None):
        self.num_classes = num_classes
        self.box_encoding_len = box_encoding_len
        if regularizer_type is None:
            assert regularizer_kwargs is None, 'No regularizer no kwargs'
        # weight regularisers only enter the training loss (models.py:283-290): accepted, unused
        self._regularizer = None
        self._layer_configs = layer_configs
        self._default_layers_type = {                                   # models.py:48-75
            'scatter_max_point_set_pooling': gnn.PointSetPooling(
                point_feature_fn=gnn.multi_layer_neural_network_fn,
                aggregation_fn=gnn.graph_scatter_max_fn,
                output_fn=gnn.multi_layer_neural_network_fn),
            'scatter_max_graph_auto_center_net': gnn.GraphNetAutoCenter(
                edge_feature_fn=gnn.multi_layer_neural_network_fn,
                aggregation_fn=gnn.graph_scatter_max_fn,
                update_fn=gnn.multi_layer_neural_network_fn,
                auto_offset_fn=gnn.multi_layer_neural_network_fn),
            'classaware_predictor': gnn.ClassAwarePredictor(
                cls_fn=partial(gnn.multi_layer_fc_fn, Ks=(64,), num_layer=2),
                loc_fn=partial(gnn.multi_layer_fc_fn, Ks=(64, 64,), num_layer=3)),
            'classaware_predictor_128': gnn.ClassAwarePredictor(
                cls_fn=partial(gnn.multi_layer_fc_fn, Ks=(128,), num_layer=2),
                loc_fn=partial(gnn.multi_layer_fc_fn, Ks=(128, 128), num_layer=3)),
            'classaware_separated_predictor': gnn.ClassAwareSeparatedPredictor(
                cls_fn=partial(gnn.multi_layer_fc_fn, Ks=(64,), num_layer=2),
                loc_fn=partial(gnn.multi_layer_fc_fn, Ks=(64, 64,), num_layer=3)),
        }
        assert mode in ['train', 'eval', 'test'], 'Unsupported mode'
        self._mode = mode
        self._store = None

    # -- weights ------------------------------------------------------------------------------
    def load_weights(self, variables):
        """variables: {tf variable name: array}, e.g. from utils.tf_checkpoint.load_checkpoint."""
        self._store = gnn.VariableStore(variables)
        return self

    def load_checkpoint(self, checkpoint_path):
        """checkpoint dir or 'dir/model-N' prefix written by the reference's tf.train.Saver."""
        return self.load_weights(tf_checkpoint.load_checkpoint(checkpoint_path))

    # -- forward ------------------------------------------------------------------------------
    @staticmethod
    def _to_device(x, dtype):
        if isinstance(x, torch.Tensor):
            t = x
            if not t.is_cuda:
                t = t.cuda()
            return t if t.dtype == dtype else t.to(dtype)
        return torch.from_numpy(np.ascontiguousarray(x)).cuda().to(dtype)

    @staticmethod
    def _stamp(t, ranges):
        """What models.graph_gen attaches to the index tensors it produces: the ranges they were built for and
        the tensor's version counter, so that an in-place edit (manual batching offsets) invalidates the stamp."""
        return tuple(int(r) for r in ranges) + (getattr(t, '_version', None),)

    def predict(self, t_initial_vertex_features, t_vertex_coord_list, t_keypoint_indices_list,
                t_edges_list, is_training=False):
        """models.py:79-163.  -> (logits [K, C], box_encodings [K, C, box_encoding_len])."""
        if self._store is None:
            raise RuntimeError('model has no weights: call load_checkpoint / load_weights first')
        numpy_io = not isinstance(t_initial_vertex_features, torch.Tensor)
        tfeatures = self._to_device(t_initial_vertex_features, torch.float32).contiguous()
        coords = [self._to_device(c, torch.float32).contiguous() for c in t_vertex_coord_list]
        keypoints = [None if k is None else self._to_device(k, torch.int32) for k in t_keypoint_indices_list]
        # Shape / range contract of the index inputs.  The reference gets these checks from TF at sess.run
        # (tf.gather and unsorted_segment_max raise InvalidArgumentError, run.py:260); here they are made ONCE
        # per predict call so that the fused kernels may skip their per-layer read-back of the error flag.
        if tfeatures.shape[0] != coords[0].shape[0]:
            raise ValueError('features have %d rows, level-0 coordinates %d' % (tfeatures.shape[0], coords[0].shape[0]))
        for level, k in enumerate(keypoints):
            if k is None or level + 1 >= len(coords):
                continue
            if k.shape[0] != coords[level + 1].shape[0]:
                raise ValueError('keypoint_indices[%d] has %d rows, level-%d coordinates %d'
                                 % (level, k.shape[0], level + 1, coords[level + 1].shape[0]))
            if getattr(t_keypoint_indices_list[level], '_pg_trusted', None) != self._stamp(
                    t_keypoint_indices_list[level], (coords[level].shape[0],)) and k.numel() > 0:
                kk = k.reshape(-1).contiguous()
                _lib.check_edges(kk, kk, coords[level].shape[0], coords[level].shape[0])
        edges = []
        trusted = []
        for level, e in enumerate(t_edges_list):
            stamp = getattr(e, '_pg_trusted', None)         # set by models.graph_gen on its own output
            ranges = (coords[level].shape[0], coords[level + 1].shape[0]) if level + 1 < len(coords) else None
            fresh = ranges is not None and stamp == self._stamp(e, ranges)
            e = self._to_device(e, torch.int32)
            if e.dim() != 2 or e.shape[1] != 2:
                raise ValueError('edges[%d] must be [E, 2] (source, destination), got %s' % (level, tuple(e.shape)))
            if e.stride(0) != 1:                 # make the (src, dst) columns contiguous
                e = e.t().contiguous().t()
            if ranges is not None and not fresh and e.shape[0] > 0:
                # foreign (or edited) edge list: one synchronising range check here
                _lib.check_edges(e[:, 0], e[:, 1], ranges[0], ranges[1])
            edges.append(e)
            trusted.append(ranges is not None)
        with gnn.variable_session(self._store):
            for idx in range(len(self._layer_configs) - 1):
                layer_config = self._layer_configs[idx]
                graph_level = layer_config['graph_level']
                with gnn.variable_scope(layer_config['scope']):
                    flgn = self._default_layers_type[layer_config['type']]
                    gnn._ctx.trusted_edges = trusted[graph_level]
                    tfeatures = flgn.apply_regular(tfeatures, coords[graph_level], keypoints[graph_level],
                                                   edges[graph_level], **layer_config['kwargs'])
            gnn._ctx.trusted_edges = False
            predictor_config = self._layer_configs[-1]
            assert predictor_config['type'] in ('classaware_predictor', 'classaware_predictor_128',
                                                'classaware_separated_predictor')
            predictor = self._default_layers_type[predictor_config['type']]
            with gnn.variable_scope(predictor_config['scope']):
                logits, box_encodings = predictor.apply_regular(
                    tfeatures, num_classes=self.num_classes, box_encoding_len=self.box_encoding_len,
                    **predictor_config['kwargs'])
        if numpy_io:
            return logits.cpu().numpy(), box_encodings.cpu().numpy()
        return logits, box_encodings

    def postprocess(self, logits):
        """models.py:165-168: softmax over classes."""
        if isinstance(logits, torch.Tensor):
            fused = getattr(logits, '_pg_probs', None)     # the predictor heads kernel already did the softmax
            if fused is not None and fused[1] == logits._version:
                return fused[0]
            return _lib.softmax_rows(logits.contiguous())
        t = torch.from_numpy(np.ascontiguousarray(logits, dtype=np.float32)).cuda()
        return _lib.softmax_rows(t).cpu().numpy()


def get_model(model_name):
    """models.py:313-319."""
    model_map = {
        'multi_layer_fast_local_graph_model_v2': MultiLayerFastLocalGraphModelV2,
    }
    return model_map[model_name]

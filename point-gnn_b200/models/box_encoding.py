"""Box codecs - the decoding half of the reference's ``models/box_encoding.py`` that inference uses
(/root/reference/models/box_encoding.py:210-229, 265-299, 345-395, 469-503), on the GPU.

``get_box_decoding_fn(name)`` / ``get_encoding_len(name)`` keep the reference's names and call
convention (run.py:100-102, 278-280).  The two codecs whose decoder takes run.py's four-argument call are
built: ``classaware_all_class_box_encoding`` (every shipped config) and
``classaware_all_class_box_canonical_encoding`` (box_encoding.py:345-395).  The three-argument decoders
(``direct``, ``center``, ``voxelnet``, ``classaware_voxelnet``) fail at run.py's first decode in the reference
and are not built.  The training-time ENCODERS (box_encoding.py:231-263, 301-343) are part of label
assignment, outside the inference path (SURVEY section 2).
"""
import numpy as np
import torch

from .. import _lib

median_object_size_map = {          # box_encoding.py:210-219: (l, h, w)
    'Cyclist': (1.76, 1.75, 0.6),
    'Van': (4.98, 2.13, 1.88),
    'Tram': (14.66, 3.61, 2.6),
    'Car': (3.88, 1.5, 1.63),
    'Misc': (2.52, 1.65, 1.51),
    'Pedestrian': (0.88, 1.77, 0.65),
    'Truck': (10.81, 3.34, 2.63),
    'Person_sitting': (0.75, 1.26, 0.59),
}


def class_table(label_map, num_classes):
    """Per class label (l, h, w, yaw offset); l <= 0 = label not decoded (Background, DontCare).
    box_encoding.py:268-291: label ``cls`` is the "horizontal" variant, ``cls + 1`` the "vertical" one."""
    table = [[-1.0, -1.0, -1.0, 0.0] for _ in range(num_classes)]
    for name, label in label_map.items():
        if name in ('Background', 'DontCare'):
            continue
        l, h, w = median_object_size_map[name]
        table[label] = [l, h, w, 0.0]
        table[label + 1] = [l, h, w, 0.5 * np.pi]
    return table


def _decode_slot0(cls_labels, points_xyz, encoded_boxes, label_map, flags):
    """The reference's four-argument decoders: slot 0 of every row decoded under that row's label, the other slots
    only offset by the point."""
    numpy_io = not isinstance(encoded_boxes, torch.Tensor)
    enc = torch.as_tensor(np.ascontiguousarray(encoded_boxes, dtype=np.float32)).cuda() if numpy_io else encoded_boxes
    xyz = torch.as_tensor(np.ascontiguousarray(points_xyz, dtype=np.float32)).cuda() if numpy_io else points_xyz
    labels = torch.as_tensor(np.asarray(cls_labels)).reshape(-1).to(enc.device)
    m, c, _ = enc.shape
    num_labels = int(max(int(labels.max()) + 2 if labels.numel() else 2, max(label_map.values()) + 2))
    table = class_table(label_map, num_labels)
    # decode slot 0 under every label, then pick per row the decoding of that row's label; other slots: offset only
    rep = enc[:, :1, :].expand(m, num_labels, 7).contiguous()
    dec = _lib.decode_boxes(rep, xyz.contiguous(), table, flags)
    out = enc.clone()
    out[:, :, :3] += xyz[:, None, :]
    out[:, 0, :] = dec[torch.arange(m, device=enc.device), labels.long().clamp(0, num_labels - 1), :]
    return out.cpu().numpy() if numpy_io else out


def classaware_all_class_box_decoding(cls_labels, points_xyz, encoded_boxes, label_map):
    """box_encoding.py:265-299.  encoded_boxes [M, C', 7] with points_xyz [M, 3]; ``cls_labels`` [M, 1] gives the
    label of slot 0 of every row (run.py:278-280 calls it with C' = 1, one row per (vertex, class) pair)."""
    return _decode_slot0(cls_labels, points_xyz, encoded_boxes, label_map, 0)


def classaware_all_class_box_canonical_decoding(cls_labels, points_xyz, encoded_boxes, label_map):
    """box_encoding.py:345-395, called as classaware_all_class_box_decoding is: x and z are (e0 l, e2 w) rotated by
    yaw' = e6 pi / 4 (l and w swapped for the "vertical" label), sizes and yaw as in the all-class rule."""
    return _decode_slot0(cls_labels, points_xyz, encoded_boxes, label_map, _lib.PG_BOX_CANONICAL)


# the codecs whose decoder the reference's run.py can call (with four arguments) -> the PG_BOX_* flag of each
DECODING_FLAGS = {
    'classaware_all_class_box_encoding': 0,
    'classaware_all_class_box_canonical_encoding': _lib.PG_BOX_CANONICAL,
}


def get_box_decoding_fn(encoding_method_name):
    """box_encoding.py:481-491."""
    decoding_method_dict = {
        'classaware_all_class_box_encoding': classaware_all_class_box_decoding,
        'classaware_all_class_box_canonical_encoding': classaware_all_class_box_canonical_decoding,
    }
    return decoding_method_dict[encoding_method_name]


def get_encoding_len(encoding_method_name):
    """box_encoding.py:493-503."""
    encoding_len_dict = {
        'direct_encoding': 7,
        'center_box_encoding': 7,
        'voxelnet_box_encoding': 7,
        'classaware_voxelnet_box_encoding': 7,
        'classaware_all_class_box_encoding': 7,
        'classaware_all_class_box_canonical_encoding': 7,
    }
    return encoding_len_dict[encoding_method_name]

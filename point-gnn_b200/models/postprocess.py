"""run.py:265-325 as one call for a batch of frames: candidate selection, box decoding and NMS / merge / rescore,
everything on the GPU (``pg_postprocess``).  ``detect`` is what the eager ``run.py`` twin (``point-gnn_b200/run.py``)
calls after ``model.predict``, and ``kitti_rows`` (run.py:361-408, ``pg_kitti_rows``) what it calls after ``detect``;
the reference-shaped single-frame entry points live in ``models.nms`` and ``models.box_encoding``."""
import torch

from .. import _lib
from . import box_encoding

LABEL_MAPS = {   # run.py:243-250
    'yaw': {'Background': 0, 'Car': 1, 'Pedestrian': 3, 'Cyclist': 5, 'DontCare': 7},
    'Car': {'Background': 0, 'Car': 1, 'DontCare': 3},
    'Pedestrian_and_Cyclist': {'Background': 0, 'Pedestrian': 1, 'Cyclist': 3, 'DontCare': 5},
}
CLASS_NAMES = {  # run.py:371-383
    'yaw': ['Background', 'Car', 'Car', 'Pedestrian', 'Pedestrian', 'Cyclist', 'Cyclist', 'DontCare'],
    'Car': ['Background', 'Car', 'Car', 'DontCare'],
    'Pedestrian_and_Cyclist': ['Background', 'Pedestrian', 'Pedestrian', 'Cyclist', 'Cyclist', 'DontCare'],
    'alpha': ['Background', 'Car', 'Car', 'Pedestrian', 'Pedestrian', 'Cyclist', 'Cyclist', 'DontCare'],
}


def decoding_flags(box_encoding_method):
    """The PG_BOX_* flag of a config's box_encoding_method.  Only the four-argument decoders run.py calls are
    built; any other name raises ValueError (the reference's run.py raises TypeError at its first decode)."""
    if box_encoding_method not in box_encoding.DECODING_FLAGS:
        raise ValueError('box_encoding_method %r: run.py decodes with (labels, xyz, boxes, label_map), which only %s '
                         'take' % (box_encoding_method, ' and '.join(sorted(box_encoding.DECODING_FLAGS))))
    return box_encoding.DECODING_FLAGS[box_encoding_method]


def detect(probs, box_encodings, last_layer_points_xyz, frame_ptr, label_method, nms_overlapped_thres,
           use_box_merge=True, use_box_score=True, want_candidates=False,
           box_encoding_method='classaware_all_class_box_encoding'):
    """probs [K, C], box_encodings [K, C, 7], last_layer_points_xyz [K, 3] (CUDA tensors, frames concatenated,
    frame_ptr [F+1] int32) -> dict of CUDA tensors: label, box [D,7], score, index (flat v*C + c), frame_ptr [F+1]
    (+ cand_index / cand_frame_ptr = run.py's box_indices when want_candidates).  box_encoding_method: the config's
    codec, which selects the decoding rule."""
    canonical = decoding_flags(box_encoding_method) == _lib.PG_BOX_CANONICAL
    num_classes = probs.shape[1]
    table = box_encoding.class_table(LABEL_MAPS[label_method], num_classes)
    if frame_ptr is None:
        frame_ptr = torch.tensor([0, probs.shape[0]], dtype=torch.int32, device=probs.device)
    return _lib.postprocess(probs.contiguous(), box_encodings.contiguous(), last_layer_points_xyz.contiguous(),
                            frame_ptr.to(torch.int32).contiguous(), table, nms_overlapped_thres,
                            merge=use_box_merge, rescore=use_box_score, want_candidates=want_candidates,
                            canonical=canonical)


def kitti_rows(det, last_layer_points_xyz, cam_to_image, num_classes, use_box_score=True):
    """run.py:361-408 on the GPU for every frame of ``det`` (``detect``'s result; with use_box_score it must have been
    called with want_candidates=True): truncation filter, 2-D boxes and occlusion rescoring (``pg_kitti_rows``).
    cam_to_image: [F,3,4] per-frame calibration (host or CUDA, converted to CUDA float64).
    -> (rows [R, 16] float64 CUDA tensor in the row layout of include/pointgnn_b200.h, row_frame_ptr [F+1] int32)."""
    dev = det['box'].device
    cti = torch.as_tensor(cam_to_image, dtype=torch.float64).to(dev).contiguous()
    cand_index = det.get('cand_index') if use_box_score else None
    cand_frame_ptr = det.get('cand_frame_ptr') if use_box_score else None
    if use_box_score and cand_index is None:
        raise ValueError('rescoring needs the candidates: call detect(..., want_candidates=True)')
    return _lib.kitti_rows(det['label'], det['box'], det['score'], det['frame_ptr'], last_layer_points_xyz.contiguous(),
                           cand_index, cand_frame_ptr, num_classes, cti, use_box_score)

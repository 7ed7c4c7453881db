"""Inference pipeline for Point-GNN on KITTI - the eager twin of the reference's ``run.py``.

Same command line, same per-frame flow, same stage timers and the same KITTI-format output files as
/root/reference/run.py; the TensorFlow-1 pieces are replaced by this package:

  reference run.py      here
  :104-150  placeholders + model.predict graph build   -> ``model = get_model(...)(...)``, nothing to build
  :192-202  tf.Session, Saver.restore                  -> ``model.load_checkpoint(CHECKPOINT_PATH)`` (no TensorFlow)
  :210-215  dataset.get_cam_points_in_image_with_rgb   -> GPU input stage (dataset.kitti_dataset, pg_cam_points_in_image)
  :219-222  graph_generate_fn(...)                     -> GPU graph build (models.graph_gen, pg_multi_level_graph)
  :252-260  sess.run(fetches, feed_dict)               -> ``model.predict`` / ``model.postprocess`` (CUDA kernels)
  :265-325  box decoding + nms.nms_boxes_3d_*          -> models.postprocess.detect (pg_postprocess), one call
  :361-433  KITTI label conversion + file writer       -> ``kitti_labels`` / ``write_kitti_file`` below (NumPy, as there)

The visualisation levels (``-l 1|2``, Open3D / OpenCV windows, run.py:151-190, 327-360, 434-473) are not part of
the detection path and are not built.  Frames keep their data on the GPU from the velodyne bytes to the kept
boxes; the only host work per frame is file I/O and the per-detection conversion to KITTI text.

    python -m pointgnn_b200.run CHECKPOINT_PATH [--test] [--no-box-merge] [--no-box-score]
           [--dataset_root_dir DIR] [--dataset_split_file FILE] [--output_dir DIR] [--precision fp32|bf16x3]
"""
import argparse
import os
import time

import numpy as np
import torch

import pointgnn_b200
from pointgnn_b200 import _lib
from pointgnn_b200.dataset import kitti_dataset
from pointgnn_b200.dataset.kitti_dataset import KittiDataset, Points
from pointgnn_b200.models import nms, postprocess
from pointgnn_b200.models.box_encoding import get_box_decoding_fn, get_encoding_len  # noqa: F401 (reference imports)
from pointgnn_b200.models.graph_gen import get_graph_generate_fn
from pointgnn_b200.models.models import get_model
from pointgnn_b200.util.config_util import load_config


def occlusion(label, xyz):
    """run.py:88-100."""
    if xyz.shape[0] == 0:
        return 0
    normals, lower, upper = kitti_dataset.box3d_to_normals(label)
    projected = np.matmul(xyz, np.transpose(normals))
    x_cover_rate = (np.max(projected[:, 0]) - np.min(projected[:, 0])) / (upper[0] - lower[0])
    y_cover_rate = (np.max(projected[:, 1]) - np.min(projected[:, 1])) / (upper[1] - lower[1])
    z_cover_rate = (np.max(projected[:, 2]) - np.min(projected[:, 2])) / (upper[2] - lower[2])
    return x_cover_rate * y_cover_rate * z_cover_rate


def input_features(config, attr):
    """run.py:225-237: the vertex features selected by config['input_features'] from attr = [i, r, g, b]."""
    kind = config['input_features']
    if kind == 'irgb':
        return attr
    if kind == '0rgb':
        return torch.cat([torch.zeros_like(attr[:, :1]), attr[:, 1:]], dim=1)
    if kind == '0000':
        return torch.zeros_like(attr)
    if kind == 'i000':
        return torch.cat([attr[:, :1], torch.zeros_like(attr[:, 1:4])], dim=1)
    if kind == 'i':
        return attr[:, :1].contiguous()
    if kind == '0':
        return torch.zeros_like(attr[:, :1])
    raise KeyError(kind)


def kitti_labels(class_labels, detection_boxes_3d, box_probs, candidate_xyz, calib, label_method, use_box_score,
                 image_size=(1242.0, 375.0)):
    """run.py:361-408: detections of one frame -> the tuples written to the KITTI result file.

    class_labels [D], detection_boxes_3d [D,7], box_probs [D] = NMS output; candidate_xyz [B,3] = the coordinates of
    ALL candidate vertices of the frame (``last_layer_points_xyz[box_indices]``, run.py:399-401) for the occlusion
    re-scoring."""
    all_class_name = postprocess.CLASS_NAMES[label_method]
    corners_all = nms.boxes_3d_to_corners(detection_boxes_3d)
    pred_labels = []
    for i in range(len(corners_all)):
        cam = np.hstack([corners_all[i], np.ones([8, 1])])
        img = np.matmul(cam, np.transpose(calib['cam_to_image']))
        corners_xy = (img / img[:, [2]])[:, :2]
        class_name = all_class_name[class_labels[i]]
        xmin, ymin = np.amin(corners_xy, axis=0)
        xmax, ymax = np.amax(corners_xy, axis=0)
        clip_xmin, clip_ymin = max(xmin, 0.0), max(ymin, 0.0)
        clip_xmax, clip_ymax = min(xmax, image_size[0]), min(ymax, image_size[1])
        truncation_rate = 1.0 - (clip_ymax - clip_ymin) * (clip_xmax - clip_xmin) / ((ymax - ymin) * (xmax - xmin))
        if truncation_rate > 0.4:
            continue
        x3d, y3d, z3d, l, h, w, yaw = detection_boxes_3d[i]
        assert l > 0, str(i)
        score = box_probs[i]
        if use_box_score:
            tmp_label = {'x3d': x3d, 'y3d': y3d, 'z3d': z3d, 'yaw': yaw, 'height': h, 'width': w, 'length': l}
            inside_mask = kitti_dataset.sel_xyz_in_box3d(tmp_label, candidate_xyz)
            score = (1 + occlusion(tmp_label, candidate_xyz[inside_mask])) * score
        pred_labels.append((class_name, -1, -1, 0, clip_xmin, clip_ymin, clip_xmax, clip_ymax, h, w, l, x3d, y3d, z3d,
                            yaw, score))
    return pred_labels


def write_kitti_file(filename, pred_labels):
    """run.py:421-429: one line per detection, fields separated (and followed) by a blank, one empty line at the end."""
    os.makedirs(os.path.dirname(filename), exist_ok=True)
    with open(filename, 'w') as f:
        for pred_label in pred_labels:
            for field in pred_label:
                f.write(str(field) + ' ')
            f.write('\n')
        f.write('\n')


def main(argv=None):
    parser = argparse.ArgumentParser(description='Point-GNN inference on KITTI (H100 twin of run.py)')
    parser.add_argument('checkpoint_path', type=str, help='Path to checkpoint')
    parser.add_argument('-l', '--level', type=int, default=0, help='Visualization level: only 0 (disabled) is built')
    parser.add_argument('--test', dest='test', action='store_true', default=False, help='Enable test model')
    parser.add_argument('--no-box-merge', dest='use_box_merge', action='store_false', default=True,
                        help='Disable box merge.')
    parser.add_argument('--no-box-score', dest='use_box_score', action='store_false', default=True,
                        help='Disable box score.')
    parser.add_argument('--dataset_root_dir', type=str, default='../dataset/kitti/',
                        help='Path to KITTI dataset. Default="../dataset/kitti/"')
    parser.add_argument('--dataset_split_file', type=str, default='',
                        help='Path to KITTI dataset split file. Default="DATASET_ROOT_DIR/3DOP_splits/val.txt"')
    parser.add_argument('--output_dir', type=str, default='',
                        help='Path to save the detection results. Default="CHECKPOINT_PATH/eval/"')
    parser.add_argument('--precision', type=str, default=None, choices=['fp32', 'bf16x3'],
                        help='Arithmetic of the dense layers (default: bf16x3 on sm_90, fp32-class accuracy)')
    args = parser.parse_args(argv)
    if args.level != 0:
        raise NotImplementedError('visualisation levels 1 / 2 (Open3D windows) are not built')
    IS_TEST = args.test
    USE_BOX_MERGE = args.use_box_merge
    USE_BOX_SCORE = args.use_box_score
    DATASET_DIR = args.dataset_root_dir
    if args.dataset_split_file == '':
        DATASET_SPLIT_FILE = os.path.join(DATASET_DIR, './3DOP_splits/val.txt')
    else:
        DATASET_SPLIT_FILE = args.dataset_split_file
    if args.output_dir == '':
        OUTPUT_DIR = os.path.join(args.checkpoint_path, './eval/')
    else:
        OUTPUT_DIR = args.output_dir
    CHECKPOINT_PATH = args.checkpoint_path
    CONFIG_PATH = os.path.join(CHECKPOINT_PATH, 'config')
    assert os.path.isfile(CONFIG_PATH), 'No config file found in %s' % CONFIG_PATH
    config = load_config(CONFIG_PATH)
    # setup dataset ===========================================================
    if IS_TEST:
        dataset = KittiDataset(
            os.path.join(DATASET_DIR, 'image/testing/image_2'),
            os.path.join(DATASET_DIR, 'velodyne/testing/velodyne/'),
            os.path.join(DATASET_DIR, 'calib/testing/calib/'),
            '',
            num_classes=config['num_classes'],
            is_training=False)
    else:
        dataset = KittiDataset(
            os.path.join(DATASET_DIR, 'image/training/image_2'),
            os.path.join(DATASET_DIR, 'velodyne/training/velodyne/'),
            os.path.join(DATASET_DIR, 'calib/training/calib/'),
            os.path.join(DATASET_DIR, 'labels/training/label_2'),
            DATASET_SPLIT_FILE,
            num_classes=config['num_classes'],
            is_training=False)       # labels are only read for visualisation in the reference; not needed here
    NUM_TEST_SAMPLE = dataset.num_files
    NUM_CLASSES = dataset.num_classes
    # setup model =============================================================
    BOX_ENCODING_LEN = get_encoding_len(config['box_encoding_method'])
    pointgnn_b200.set_precision(args.precision or ('bf16x3' if _lib.tc_available() else 'fp32'))
    model = get_model(config['model_name'])(num_classes=NUM_CLASSES, box_encoding_len=BOX_ENCODING_LEN, mode='test',
                                            **config['model_kwargs'])
    print('Restore from checkpoint %s' % CHECKPOINT_PATH)
    model.load_checkpoint(CHECKPOINT_PATH)
    graph_generate_fn = get_graph_generate_fn(config['graph_gen_method'])
    device = torch.device('cuda', torch.cuda.current_device())
    # running network =========================================================
    time_dict = {}
    for frame_idx in range(0, NUM_TEST_SAMPLE):
        start_time = time.time()
        # provide input ======================================================
        calib = dataset.get_calib(frame_idx)
        image = dataset.get_image(frame_idx)
        want_rgb = config['input_features'] in ('irgb', '0rgb')
        xyz, attr, _ = kitti_dataset.cam_points_in_image_batch(
            [dataset.get_velo_data(frame_idx)], [calib], [(image.shape[1], image.shape[0])],
            [image] if want_rgb else None, device=device)
        if not want_rgb and config['input_features'] in ('0000', 'i000'):
            attr = torch.cat([attr, torch.zeros((attr.shape[0], 3), device=device)], dim=1)
        torch.cuda.synchronize()
        input_time = time.time()
        time_dict['fetch input'] = time_dict.get('fetch input', 0) + input_time - start_time
        (vertex_coord_list, keypoint_indices_list, edges_list) = graph_generate_fn(
            xyz, **config['runtime_graph_gen_kwargs'])
        torch.cuda.synchronize()
        graph_time = time.time()
        time_dict['gen graph'] = time_dict.get('gen graph', 0) + graph_time - input_time
        input_v = input_features(config, attr)
        last_layer_graph_level = config['model_kwargs']['layer_configs'][-1]['graph_level']
        last_layer_points_xyz = vertex_coord_list[last_layer_graph_level + 1]
        # run forwarding =====================================================
        logits, pred_box = model.predict(input_v, vertex_coord_list, keypoint_indices_list, edges_list, is_training=True)
        probs = model.postprocess(logits)
        torch.cuda.synchronize()
        gnn_time = time.time()
        time_dict['gnn inference'] = time_dict.get('gnn inference', 0) + gnn_time - graph_time
        # box decoding + nms ==================================================
        det = postprocess.detect(probs, pred_box, last_layer_points_xyz, None, config['label_method'],
                                 config['nms_overlapped_thres'], use_box_merge=USE_BOX_MERGE,
                                 use_box_score=USE_BOX_SCORE, want_candidates=True)
        class_labels = det['label'].cpu().numpy()
        detection_boxes_3d = det['box'].cpu().numpy()
        box_probs = det['score'].cpu().numpy()
        cand_vertices = (det['cand_index'] // NUM_CLASSES).long()
        candidate_xyz = last_layer_points_xyz[cand_vertices].cpu().numpy()
        decode_time = time.time()
        time_dict['decode box'] = time_dict.get('decode box', 0) + decode_time - gnn_time
        pred_labels = []
        if len(class_labels) > 0:
            # convert to KITTI ================================================
            pred_labels = kitti_labels(class_labels, detection_boxes_3d, box_probs, candidate_xyz, calib,
                                       config['label_method'], USE_BOX_SCORE)
        nms_time = time.time()
        time_dict['nms'] = time_dict.get('nms', 0) + nms_time - decode_time
        # output ===========================================================
        filename = OUTPUT_DIR + '/data/' + dataset.get_filename(frame_idx) + '.txt'
        write_kitti_file(filename, pred_labels)
        total_time = time.time()
        time_dict['total'] = time_dict.get('total', 0) + total_time - start_time
    # time statics ============================================================
    for key in time_dict:
        print(key + ' time : ' + str(time_dict[key] / max(NUM_TEST_SAMPLE, 1)))
    return time_dict


if __name__ == '__main__':
    main()

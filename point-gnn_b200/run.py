"""Inference pipeline for Point-GNN on KITTI - the eager twin of the reference's ``run.py``.

Same command line, same stage timers and the same KITTI-format output files as /root/reference/run.py; the
TensorFlow-1 pieces are replaced by this package:

  reference run.py      here
  :104-150  placeholders + model.predict graph build   -> ``model = get_model(...)(...)``, nothing to build
  :192-202  tf.Session, Saver.restore                  -> ``model.load_checkpoint(CHECKPOINT_PATH)`` (no TensorFlow)
  :210-215  dataset.get_cam_points_in_image_with_rgb   -> GPU input stage (dataset.kitti_dataset, pg_cam_points_in_image;
                                                          with config['downsample_by_voxel_size']: pg_velo_to_cam,
                                                          pg_voxel_average, pg_cam_points_crop)
  :219-222  graph_generate_fn(...)                     -> GPU graph build (models.graph_gen, pg_multi_level_graph)
  :252-260  sess.run(fetches, feed_dict)               -> ``model.predict`` / ``model.postprocess`` (CUDA kernels)
  :265-325  box decoding + nms.nms_boxes_3d_*          -> models.postprocess.detect (pg_postprocess), one call
  :361-408  KITTI label conversion                     -> models.postprocess.kitti_rows (pg_kitti_rows), one call;
                                                          ``kitti_labels`` below is the NumPy form, kept as the reference
  :421-433  file writer                                -> ``write_kitti_file`` below

The visualisation levels (``-l 1|2``, Open3D / OpenCV windows, run.py:151-190, 327-360, 434-473) are not part of
the detection path and are not built.

Batches.  ``--batch_size N`` (default 1) groups consecutive frames of the split; the last batch may be shorter.
Every stage takes the whole batch in one call (indices are global, frames are independent), so the files do not
depend on N.  While the GPU runs batch i, a worker thread reads batch i+2's files (velodyne .bin, calibration, and
the image - only its size, from the PNG header, when the input features use no colour), and the input stage and
graph build of batch i+1 are issued on the ``utils.prefetch.GraphPrefetcher`` side stream.  Per batch the host then
waits for the forward pass, runs ``detect`` and ``kitti_rows`` and reads the rows back once; what is left is the text
formatting and the file writes.

Timers (run.py's names, per-frame means: the sum over batches divided by the number of frames).  Stages of different
batches overlap, so each timer is the host time spent in its step, and a GPU stage that overlaps another one is
charged to the step whose wait it ends:
  fetch input    waiting for the worker thread's files of the batch and issuing its input stage (one size read-back
                 on the side stream)
  gen graph      issuing the batch's graph build on the side stream (its one size read-back included)
  gnn inference  issuing the forward pass and then waiting for it, after the next batch's input and graph have been
                 issued
  decode box     ``detect``: box decoding and NMS, ending in its read-back of the number of kept boxes
  nms            ``kitti_rows``, the one read-back of the rows and their conversion to KITTI tuples (run.py's label
                 conversion, which its ``nms`` timer covers)
  total          wall time of the whole loop, file writes included, divided by the number of frames

Processes.  ``--processes N`` (default 1) runs the split in N spawned worker processes: rank r takes positions
r, r + N, r + 2N, ... of the split (``rank_batches``), batches them ``--batch_size`` at a time and runs them on device
``r % torch.cuda.device_count()``, so ``CUDA_VISIBLE_DEVICES`` picks the devices and N above the device count puts
several ranks on one device, whose host work then overlaps.  Each rank has its own reader thread, graph prefetcher,
model and prepared layers and writes its own frames' files; the files are those of one process.  The parent checks
the command line, the config and the split before it spawns anything, prints the timers of the whole job (each stage
summed over the ranks, ``total`` the slowest rank's loop) and returns them.  A rank that raises, or a Ctrl-C, stops
every rank before ``main`` raises.  With N = 1 nothing is spawned: the run happens in the calling process.

    python -m pointgnn_b200.run CHECKPOINT_PATH [--test] [--no-box-merge] [--no-box-score]
           [--dataset_root_dir DIR] [--dataset_split_file FILE] [--output_dir DIR] [--precision fp32|bf16x3|fp16]
           [--batch_size N] [--processes N]
"""
import argparse
import multiprocessing
import os
import queue
import signal
import time
import traceback
from concurrent.futures import ThreadPoolExecutor

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
from pointgnn_b200.utils.prefetch import GraphPrefetcher
from pointgnn_b200.utils.sharding import frames_for_rank


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


def input_stage(config, velo, calib, size, image, device):
    """run.py:210-215 for a batch: the frames' camera-frame points inside their images, averaged per voxel first when
    config['downsample_by_voxel_size'] is set (absent or null: off) -> (xyz, attr, frame_ptr) on the device, attr
    padded to four columns for the input features that want them without colour."""
    xyz, attr, frame_ptr = kitti_dataset.cam_points_in_image_batch(
        velo, calib, size, image, device=device, downsample_voxel_size=config.get('downsample_by_voxel_size'))
    if image is None and config['input_features'] in ('0000', 'i000'):
        attr = torch.cat([attr, torch.zeros((attr.shape[0], 3), device=device)], dim=1)
    return xyz, attr, frame_ptr


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


def kitti_labels_from_rows(rows, num_frames, label_method):
    """The rows of ``postprocess.kitti_rows`` (read back as a NumPy [R, 16] float64 array) -> one list per frame of the
    tuples ``kitti_labels`` returns, with the same field types, so that ``write_kitti_file`` prints the same text:
    h, w, l, x, y, z, yaw as float32, the clipped box as float64, the score as float64 when rescoring found candidates
    inside the box and as the float32 NMS score otherwise (run.py:406 multiplies by the Python int 1 then)."""
    all_class_name = postprocess.CLASS_NAMES[label_method]
    per_frame = [[] for _ in range(num_frames)]
    box = rows[:, 3:10].astype(np.float32)          # exact: the kernel widened these float32 values
    for r in range(rows.shape[0]):
        row = rows[r]
        x3d, y3d, z3d, l, h, w, yaw = box[r]
        clip_xmin, clip_ymin, clip_xmax, clip_ymax = (np.float64(v) for v in row[10:14])
        score = np.float64(row[14]) if row[15] > 0 else np.float32(row[14])
        per_frame[int(row[1])].append((all_class_name[int(row[2])], -1, -1, 0, clip_xmin, clip_ymin, clip_xmax,
                                       clip_ymax, h, w, l, x3d, y3d, z3d, yaw, score))
    return per_frame


def write_kitti_file(filename, pred_labels):
    """run.py:421-429: one line per detection, fields separated (and followed) by a blank, one empty line at the end."""
    os.makedirs(os.path.dirname(filename), exist_ok=True)
    with open(filename, 'w') as f:
        for pred_label in pred_labels:
            for field in pred_label:
                f.write(str(field) + ' ')
            f.write('\n')
        f.write('\n')


def open_job(args):
    """What ``main`` reads and checks before the first frame: the config (its codec must be one run.py decodes) and
    the split -> (config, dataset, output directory)."""
    IS_TEST = args.test
    DATASET_DIR = args.dataset_root_dir
    if args.dataset_split_file == '':
        DATASET_SPLIT_FILE = os.path.join(DATASET_DIR, './3DOP_splits/val.txt')
    else:
        DATASET_SPLIT_FILE = args.dataset_split_file
    if args.output_dir == '':
        OUTPUT_DIR = os.path.join(args.checkpoint_path, './eval/')
    else:
        OUTPUT_DIR = args.output_dir
    CONFIG_PATH = os.path.join(args.checkpoint_path, 'config')
    assert os.path.isfile(CONFIG_PATH), 'No config file found in %s' % CONFIG_PATH
    config = load_config(CONFIG_PATH)
    # the decoding rule of the model's box codec; a codec run.py cannot decode fails here, before any frame is read
    postprocess.decoding_flags(config['box_encoding_method'])
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
    return config, dataset, OUTPUT_DIR


def run_batches(args, config, dataset, output_dir, batches):
    """Run ``batches`` (lists of positions in the split) on the current device and write their files -> the timers'
    sums in seconds.  The work of one process: ``main`` calls it in-process, each rank of ``--processes`` in its
    worker."""
    USE_BOX_MERGE = args.use_box_merge
    USE_BOX_SCORE = args.use_box_score
    OUTPUT_DIR = output_dir
    NUM_CLASSES = dataset.num_classes
    # setup model =============================================================
    BOX_ENCODING_LEN = get_encoding_len(config['box_encoding_method'])
    pointgnn_b200.set_precision(args.precision or ('bf16x3' if _lib.tc_available() else 'fp32'))
    model = get_model(config['model_name'])(num_classes=NUM_CLASSES, box_encoding_len=BOX_ENCODING_LEN, mode='test',
                                            **config['model_kwargs'])
    print('Restore from checkpoint %s' % args.checkpoint_path)
    model.load_checkpoint(args.checkpoint_path)
    graph_generate_fn = get_graph_generate_fn(config['graph_gen_method'])
    device = torch.device('cuda', torch.cuda.current_device())
    # running network =========================================================
    time_dict = {}

    def charge(key, seconds):
        time_dict[key] = time_dict.get(key, 0) + seconds

    want_rgb = config['input_features'] in ('irgb', '0rgb')
    last_layer_graph_level = config['model_kwargs']['layer_configs'][-1]['graph_level']

    def read_files(frames):
        """Host file work of one batch (worker thread): velodyne, calibration, image or only its size."""
        velo, calib, size, image = [], [], [], []
        for frame_idx in frames:
            velo.append(dataset.get_velo_data(frame_idx))
            calib.append(dataset.get_calib(frame_idx))
            if want_rgb:
                image.append(dataset.get_image(frame_idx))
                size.append(image[-1].shape[:2])
            else:
                size.append(dataset.get_image_size(frame_idx))
        return velo, calib, [(w, h) for h, w in size], image if want_rgb else None

    reader = ThreadPoolExecutor(max_workers=1)
    pending = {}

    def start_reading(b):
        if b < len(batches):
            pending[b] = reader.submit(read_files, batches[b])

    prefetcher = GraphPrefetcher(graph_generate_fn, config['runtime_graph_gen_kwargs'], device)

    def issue(b):
        """Input stage + graph build of batch b on the prefetcher's side stream -> (graph ticket, calibrations)."""
        t0 = time.time()
        velo, calib, size, image = pending.pop(b).result()
        start_reading(b + 1)
        with torch.cuda.stream(prefetcher.stream):
            xyz, attr, frame_ptr = input_stage(config, velo, calib, size, image, device)
            t1 = time.time()
            # submitted from the side stream: the inputs were made there, so the build waits for nothing else
            ticket = prefetcher.submit(xyz, attr, frame_ptr)
        charge('fetch input', t1 - t0)
        charge('gen graph', time.time() - t1)
        return ticket, calib

    try:
        start_time = time.time()
        start_reading(0)
        upcoming = issue(0) if batches else None
        for b, frames in enumerate(batches):
            ticket, calib = upcoming
            t0 = time.time()
            attr, vertex_coord_list, keypoint_indices_list, edges_list = prefetcher.collect(ticket)
            input_v = input_features(config, attr)
            last_layer_points_xyz = vertex_coord_list[last_layer_graph_level + 1]
            # run forwarding =================================================
            logits, pred_box = model.predict(input_v, vertex_coord_list, keypoint_indices_list, edges_list,
                                             is_training=True)
            probs = model.postprocess(logits)
            gnn_issue = time.time() - t0
            if b + 1 < len(batches):
                upcoming = issue(b + 1)
            t1 = time.time()
            torch.cuda.current_stream().synchronize()
            t2 = time.time()
            charge('gnn inference', gnn_issue + t2 - t1)
            # box decoding + nms =============================================
            det = postprocess.detect(probs, pred_box, last_layer_points_xyz,
                                     ticket.frame_ptrs[last_layer_graph_level + 1], config['label_method'],
                                     config['nms_overlapped_thres'], use_box_merge=USE_BOX_MERGE,
                                     use_box_score=USE_BOX_SCORE, want_candidates=USE_BOX_SCORE,
                                     box_encoding_method=config['box_encoding_method'])
            t3 = time.time()
            charge('decode box', t3 - t2)
            # convert to KITTI ===============================================
            rows, _ = postprocess.kitti_rows(det, last_layer_points_xyz, np.stack([c['cam_to_image'] for c in calib]),
                                             NUM_CLASSES, USE_BOX_SCORE)
            pred_labels = kitti_labels_from_rows(rows.cpu().numpy(), len(frames), config['label_method'])
            charge('nms', time.time() - t3)
            # output =========================================================
            for frame_idx, labels in zip(frames, pred_labels):
                write_kitti_file(OUTPUT_DIR + '/data/' + dataset.get_filename(frame_idx) + '.txt', labels)
            # the ticket's tensors were made on the side stream; they are released only now that batch b is done
            del ticket
        if batches:
            charge('total', time.time() - start_time)
    finally:
        reader.shutdown(wait=True, cancel_futures=True)
    return time_dict


def rank_batches(num_frames, batch_size, rank, world):
    """Batches of rank ``rank`` of ``world``: its positions in the split (``frames_for_rank``: rank, rank + world,
    ...) cut ``batch_size`` at a time, the last batch possibly shorter.  World 1 gives consecutive frames."""
    frames = frames_for_rank(num_frames, rank, world)
    return [frames[first:first + batch_size] for first in range(0, len(frames), batch_size)]


def merge_rank_times(per_rank):
    """The ranks' timer sums, in rank order -> the job's: each stage summed over the ranks, ``total`` the slowest
    rank's loop, so that frames / total is the job's frames/s."""
    merged = {}
    for times in per_rank:
        for key, seconds in times.items():
            merged[key] = max(merged.get(key, 0), seconds) if key == 'total' else merged.get(key, 0) + seconds
    return merged


def _rank_main(args, rank, device, deterministic, results):
    """Worker process of rank ``rank``: its batches on ``device`` -> ('done', rank, timers) or ('failed', rank,
    traceback text) on ``results``.  A rank without frames loads nothing and reports no time."""
    # the parent alone answers Ctrl-C, by stopping every rank
    signal.signal(signal.SIGINT, signal.SIG_IGN)
    try:
        # a spawned interpreter starts with the switch off; turn it on as the caller had it (only then: the call
        # imports torch._inductor, seconds of start-up)
        if deterministic[0]:
            torch.use_deterministic_algorithms(True, warn_only=deterministic[1])
        config, dataset, output_dir = open_job(args)
        batches = rank_batches(dataset.num_files, args.batch_size, rank, args.processes)
        time_dict = {}
        if batches:
            torch.cuda.set_device(device)
            time_dict = run_batches(args, config, dataset, output_dir, batches)
        results.put(('done', rank, time_dict))
    except BaseException:
        results.put(('failed', rank, traceback.format_exc()))


def run_ranks(args):
    """Run the ``args.processes`` ranks in spawned processes (CUDA cannot be forked), rank r on device
    r % device count -> ``merge_rank_times`` of their timers.  If a rank fails, or on Ctrl-C, every rank is stopped
    and waited for before the exception, which names the failing rank and carries its traceback, propagates."""
    devices = torch.cuda.device_count()
    if devices == 0:
        raise RuntimeError('point-gnn_b200 needs a CUDA device (no CPU fallback)')
    world = args.processes
    deterministic = (torch.are_deterministic_algorithms_enabled(),
                     torch.is_deterministic_algorithms_warn_only_enabled())
    context = multiprocessing.get_context('spawn')
    results = context.Queue()
    started, done, finished = [], {}, False
    try:
        for rank in range(world):
            proc = context.Process(target=_rank_main, args=(args, rank, rank % devices, deterministic, results),
                                   name='pointgnn_b200.run rank %d' % rank)
            proc.start()
            started.append(proc)
        while len(done) < world:
            try:
                status, rank, payload = results.get(timeout=1.0)
            except queue.Empty:
                # a rank reports before it returns, so a non-zero exit code without a report is a crash
                for r, proc in enumerate(started):
                    if r not in done and proc.exitcode not in (None, 0):
                        raise RuntimeError('run.py rank %d of %d exited with code %d without a report'
                                           % (r, world, proc.exitcode))
                continue
            if status == 'failed':
                raise RuntimeError('run.py rank %d of %d failed:\n%s' % (rank, world, payload))
            done[rank] = payload
        finished = True
    finally:
        for proc in started:
            if not finished:
                proc.terminate()
        for proc in started:
            proc.join(None if finished else 30)
            if proc.is_alive():
                proc.kill()
                proc.join()
        results.close()
    return merge_rank_times([done[rank] for rank in range(world)])


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
    parser.add_argument('--precision', type=str, default=None, choices=['fp32', 'bf16x3', 'fp16'],
                        help='Arithmetic of the dense layers (default: bf16x3 on sm_90, fp32-class accuracy; fp16: '
                             'one FP16 tensor-core pass, ~1e-2 on logits)')
    parser.add_argument('--batch_size', type=int, default=1,
                        help='Frames per forward pass (consecutive frames of the split, or of a rank\'s share of it '
                             'with --processes; default 1)')
    parser.add_argument('--processes', type=int, default=1,
                        help='Worker processes, frames sharded round-robin over them; rank r runs on device '
                             'r %% torch.cuda.device_count() (default 1: run in this process, spawn nothing)')
    args = parser.parse_args(argv)
    if args.batch_size < 1:
        parser.error('--batch_size must be >= 1, got %d' % args.batch_size)
    if args.processes < 1:
        parser.error('--processes must be >= 1, got %d' % args.processes)
    if args.level != 0:
        raise NotImplementedError('visualisation levels 1 / 2 (Open3D windows) are not built')
    config, dataset, output_dir = open_job(args)
    NUM_TEST_SAMPLE = dataset.num_files
    if args.processes == 1:
        time_dict = run_batches(args, config, dataset, output_dir,
                                rank_batches(NUM_TEST_SAMPLE, args.batch_size, 0, 1))
    else:
        time_dict = run_ranks(args)
    # time statics ============================================================
    for key in time_dict:
        print(key + ' time : ' + str(time_dict[key] / max(NUM_TEST_SAMPLE, 1)))
    return time_dict


if __name__ == '__main__':
    main()

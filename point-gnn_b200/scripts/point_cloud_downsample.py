"""Twin of the reference's ``scripts/point_cloud_downsample.py``: simulate a sparser LiDAR by keeping every
``downsample_rate``-th beam of each velodyne frame of a split, and write the result as a new velodyne tree.

    python -m pointgnn_b200.scripts.point_cloud_downsample --dataset_root_dir DIR [--dataset_split_file F]
        [--downsample_rate 2] [--num_clusters 64] [--output_dir D] [--batch_size N]

The defaults are the reference's constants and paths: the frames of ``DIR/3DOP_splits/val.txt`` read from
``DIR/velodyne/training/velodyne/``, 64 clusters, rate 2, output to
``DIR/velodyne/training_downsampled_<rate>/velodyne/<frame>.bin``.  To run a detector on the sparser data, point
``run.py``'s ``--dataset_root_dir`` at a tree whose ``velodyne/training/velodyne`` is that output.

What matches the reference exactly, given the same cluster centres: each point's zenith cosine (its float32 /
float64 dtype chain), the beam bands, the kept rows in their original order and the file bytes
(``pg_beam_downsample``, ``csrc/pg_beam.cu``).  What does not: the reference clusters the cosines with an unseeded
scikit-learn ``KMeans``, a random local optimum, so no output can match it run for run.  Here the centres are
the group means of the exact optimal 1-D partition (ties to the smallest split index), which is deterministic and
whose inertia is never above that of any ``KMeans`` fit.  Points with a zero norm (a NaN cosine in the
reference) are never kept and are not clustered; a frame with at least one but fewer clusterable points than
clusters raises ``ValueError`` naming the frame, as ``KMeans`` does.

Frames run in batches of ``--batch_size`` on the GPU, one call per batch; a worker thread reads the next batch's
files while the current one runs.  Only the velodyne files are read (the dataset constructor checks, as the
reference's does, that each frame's image and calibration exist).  The output does not depend on the batch size.
"""
import argparse
import os
import re
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from pointgnn_b200.dataset.kitti_dataset import KittiDataset, beam_downsample_batch


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description='Keep every downsample_rate-th LiDAR beam of a KITTI split (GPU)')
    parser.add_argument('--dataset_root_dir', type=str, default='../dataset/kitti/',
                        help='Path to KITTI dataset. Default="../dataset/kitti/"')
    parser.add_argument('--dataset_split_file', type=str, default='',
                        help='Path to KITTI dataset split file. Default="DATASET_ROOT_DIR/3DOP_splits/val.txt"')
    parser.add_argument('--downsample_rate', type=int, default=2, help='Keep every N-th beam band (default 2)')
    parser.add_argument('--num_clusters', type=int, default=64, help='Number of beams to cluster (default 64)')
    parser.add_argument('--output_dir', type=str, default='',
                        help='Default="DATASET_ROOT_DIR/velodyne/training_downsampled_<rate>/velodyne/"')
    parser.add_argument('--batch_size', type=int, default=8, help='Frames per GPU call (default 8)')
    args = parser.parse_args(argv)
    if args.downsample_rate < 1:
        parser.error('--downsample_rate must be >= 1, got %d' % args.downsample_rate)
    if args.num_clusters < 1:
        parser.error('--num_clusters must be >= 1, got %d' % args.num_clusters)
    if args.batch_size < 1:
        parser.error('--batch_size must be >= 1, got %d' % args.batch_size)
    if args.dataset_split_file == '':
        args.dataset_split_file = os.path.join(args.dataset_root_dir, '3DOP_splits/val.txt')
    if args.output_dir == '':
        args.output_dir = os.path.join(args.dataset_root_dir,
                                       'velodyne/training_downsampled_%d/velodyne/' % args.downsample_rate)
    return args


def main(argv=None):
    args = parse_args(argv)
    root = args.dataset_root_dir
    dataset = KittiDataset(os.path.join(root, 'image/training/image_2'), os.path.join(root, 'velodyne/training/velodyne/'),
                           os.path.join(root, 'calib/training/calib/'), '', args.dataset_split_file, is_training=False)
    device = torch.device('cuda', torch.cuda.current_device())
    num_files = dataset.num_files
    batches = [list(range(first, min(first + args.batch_size, num_files)))
               for first in range(0, num_files, args.batch_size)]
    os.makedirs(args.output_dir, exist_ok=True)
    reader = ThreadPoolExecutor(max_workers=1)
    pending = {}

    def start_reading(b):
        if b < len(batches):
            pending[b] = reader.submit(lambda frames: [dataset.get_velo_data(i) for i in frames], batches[b])

    kept_points = total_points = 0
    t0 = time.time()
    try:
        start_reading(0)
        for b, frames in enumerate(batches):
            velo_list = pending.pop(b).result()
            start_reading(b + 1)
            sizes = [v.shape[0] for v in velo_list]
            fp = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
            velo = torch.from_numpy(np.ascontiguousarray(np.vstack(velo_list), dtype=np.float32)).to(device)
            try:
                res = beam_downsample_batch(velo, torch.from_numpy(fp).to(device), args.downsample_rate,
                                            args.num_clusters)
            except ValueError as e:   # the message names the frame by its place in the batch
                m = re.search(r'frame (\d+) has', str(e))
                name = dataset.get_filename(frames[int(m.group(1))]) if m else '?'
                raise ValueError('frame %s: %s' % (name, e)) from e
            kept = res['velo'].cpu().numpy()
            out_fp = res['frame_ptr'].cpu().numpy()
            for f, frame_idx in enumerate(frames):
                kept[out_fp[f]:out_fp[f + 1]].tofile(os.path.join(args.output_dir, dataset.get_filename(frame_idx) + '.bin'))
            kept_points += int(out_fp[-1])
            total_points += int(fp[-1])
    finally:
        reader.shutdown(wait=True, cancel_futures=True)
    print('%d frames, %d of %d points kept, %.2f s -> %s' % (num_files, kept_points, total_points, time.time() - t0,
                                                             args.output_dir))
    return dict(frames=num_files, kept_points=kept_points, total_points=total_points)


if __name__ == '__main__':
    main()

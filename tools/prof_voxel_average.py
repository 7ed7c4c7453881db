"""Cost and effect of `downsample_by_voxel_size`: CUDA-event times of pg_voxel_average and of the whole input stage
with and without it, and frames/s of ``python -m pointgnn_b200.run`` with the key off and set.

Part 1, kernels: FRAMES velodyne frames of POINTS points each (oracle/synth.py full-360 frames mapped to velodyne
coordinates, so the camera crop keeps the share it keeps on KITTI), already on the device.  After WARMUP untimed
calls, each of REPEATS rounds times one call of every variant between two CUDA events, alternating the variants; the
median, minimum and maximum over the rounds are printed.  Each call ends in its own host read-back of the result
size, which the events include.

Part 2, driver: a synthetic KITTI tree and checkpoint as tools/prof_run.py makes them, one checkpoint directory per
voxel size whose ``config`` carries the key; ``run.main`` is timed for each, alternating, after one untimed run of
each.  Prints one JSON line per measurement, and the GPU's name, power limit and maximum SM clock.

    python tools/prof_voxel_average.py [--frames 8] [--points 120000] [--voxel_sizes 0.1 0.2] [--repeats 9]
                                       [--run_frames 64] [--run_points 20000] [--run_repeats 3] [--batch_size 8]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))


def kernel_times(args, conditions):
    import torch
    from oracle import synth
    from pointgnn_b200 import _lib
    from pointgnn_b200.dataset import kitti_dataset
    calib = kitti_dataset.parse_calib(os.path.join(ROOT, 'tests', 'golden', 'kitti_calib.txt'))
    velo = []
    for f in range(args.frames):
        xyz, intensity = synth.lidar_frame(2000 + f, args.points, full_360=True)
        v = np.matmul(np.hstack([xyz.astype(np.float64), np.ones([len(xyz), 1])]), np.transpose(calib['cam_to_velo']))[:, :3]
        velo.append(np.hstack([v, intensity]).astype(np.float32))
    fp = torch.from_numpy(np.concatenate([[0], np.cumsum([len(v) for v in velo])]).astype(np.int32)).cuda()
    velo = torch.from_numpy(np.vstack(velo)).cuda()
    vtc = np.stack([calib['velo_to_cam'].astype(np.float32)] * args.frames)
    cti = np.stack([calib['cam_to_image']] * args.frames)
    wh = np.array([(1242, 375)] * args.frames, np.int32)
    cam, refl = _lib.velo_to_cam(velo, fp, vtc)
    sizes = {}

    def stage(voxel_size):
        if voxel_size is None:
            out = _lib.cam_points_in_image(velo, fp, vtc, cti, wh)
        else:
            a_xyz, a_refl, a_fp = _lib.voxel_average(*_lib.velo_to_cam(velo, fp, vtc), fp, voxel_size)
            sizes['voxels', voxel_size] = a_xyz.shape[0]
            out = _lib.cam_points_crop(a_xyz, a_refl, a_fp, cti, wh)
        sizes['in image', voxel_size] = out[0].shape[0]

    variants = {'input stage, off': lambda: stage(None)}
    for vs in args.voxel_sizes:
        variants['pg_voxel_average %g' % vs] = lambda vs=vs: _lib.voxel_average(cam, refl, fp, vs)
        variants['input stage, %g' % vs] = lambda vs=vs: stage(vs)
    for _ in range(args.warmup):
        for fn in variants.values():
            fn()
    ms = {name: [] for name in variants}
    for _ in range(args.repeats):
        for name, fn in variants.items():
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            fn()
            end.record()
            end.synchronize()
            ms[name].append(start.elapsed_time(end))
    for name, t in ms.items():
        print(json.dumps({'what': name, 'frames': args.frames, 'points_per_frame': args.points,
                          'ms_median': float(np.median(t)), 'ms_min': min(t), 'ms_max': max(t), 'repeats': len(t),
                          'gpu': conditions}), flush=True)
    print(json.dumps({'what': 'sizes', 'points': int(velo.shape[0]),
                      **{'%s, %s' % (k, 'off' if vs is None else '%g' % vs): n for (k, vs), n in sizes.items()}}), flush=True)


def driver_rates(args, conditions):
    import prof_run
    from oracle import kitti as ok
    from pointgnn_b200 import run
    tmp = tempfile.mkdtemp(prefix='prof_voxel_average_')
    try:
        root = os.path.join(tmp, 'kitti')
        ok.write_synthetic_kitti(root, list(range(1000, 1000 + args.run_frames)), args.run_points)
        ckpts = {}
        for vs in [None] + list(args.voxel_sizes):
            ckpts[vs] = os.path.join(tmp, 'ckpt_%s' % vs)
            prof_run.make_checkpoint(ckpts[vs])
            with open(os.path.join(ckpts[vs], 'config')) as f:
                config = json.load(f)
            config['downsample_by_voxel_size'] = vs
            with open(os.path.join(ckpts[vs], 'config'), 'w') as f:
                json.dump(config, f)

        def once(vs):
            return run.main([ckpts[vs], '--test', '--dataset_root_dir', root, '--output_dir', os.path.join(tmp, 'out'),
                             '--batch_size', str(args.batch_size)])

        for vs in ckpts:
            once(vs)
        for rep in range(args.run_repeats):
            for vs in ckpts:
                times = once(vs)
                print(json.dumps({'what': 'run.py', 'downsample_by_voxel_size': vs, 'batch_size': args.batch_size,
                                  'repeat': rep, 'frames': args.run_frames, 'points': args.run_points,
                                  'frames_per_s': args.run_frames / times['total'],
                                  'stage_ms_per_frame': {k: 1e3 * v / args.run_frames for k, v in times.items()},
                                  'gpu': conditions}), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--frames', type=int, default=8)
    ap.add_argument('--points', type=int, default=120000)
    ap.add_argument('--voxel_sizes', type=float, nargs='+', default=[0.1, 0.2])
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--repeats', type=int, default=9)
    ap.add_argument('--run_frames', type=int, default=64)
    ap.add_argument('--run_points', type=int, default=20000)
    ap.add_argument('--run_repeats', type=int, default=3)
    ap.add_argument('--batch_size', type=int, default=8)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('prof_voxel_average.py measures on a GPU; none is present')
    import prof_run
    conditions = prof_run.gpu_conditions()
    kernel_times(args, conditions)
    if args.run_frames > 0:
        driver_rates(args, conditions)


if __name__ == '__main__':
    main()

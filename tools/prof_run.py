"""Frames/s of ``python -m pointgnn_b200.run`` end to end: file reads, GPU stages, KITTI text and file writes.

Writes a synthetic KITTI tree (oracle.kitti.write_synthetic_kitti: KITTI-sized 1242 x 375 PNGs of noise, which
decode at least as slowly as photos) and a checkpoint (the car_auto_T3_train weights with the object-class logit
biases raised by 7, as in the end-to-end tests, so that every frame has detections to convert), then times
``run.main`` for each RUN = MODULE:BATCH_SIZE and each count P of ``--processes``, alternating the runs REPEATS times
after one untimed warm-up of each.  Prints one JSON line per timed run (frames/s from run.py's ``total`` timer, the
six stage means in ms per frame, the wall time of the whole ``main`` call, worker start-up and model loads included)
and the name, power limit and maximum SM clock of the box's GPUs, with the number of CUDA devices the run sees
(``CUDA_VISIBLE_DEVICES``).  With P above that number, several ranks share a device.

    python tools/prof_run.py [--frames 64] [--points 20000] [--repeats 3] [--runs pointgnn_b200.run:1 pointgnn_b200.run:8]
                             [--processes 1 2 4]

A module other than pointgnn_b200.run is imported the same way, so an older run.py copied into the package can be
timed alternately with the current one; batch size 1 is run without the --batch_size flag, and one process without
--processes.  With several processes the stage means are the sums over the ranks (run.py's timers), and frames/s is
the frames over the slowest rank's loop.
"""
import argparse
import importlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CFG = 'car_auto_T3_train'


def gpu_conditions():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True)
    return out.stdout.strip() if out.returncode == 0 else 'unknown (nvidia-smi failed)'


def make_checkpoint(path):
    golden = os.path.join(ROOT, 'tests', 'golden')
    os.makedirs(path)
    shutil.copy(os.path.join(golden, 'config_%s.json' % CFG), os.path.join(path, 'config'))
    w = dict(np.load(os.path.join(golden, 'weights_%s.npz' % CFG)))
    b = w['output/predictor/cls/fully_connected_1/biases'].copy()
    b[1:-1] += 7.0
    w['output/predictor/cls/fully_connected_1/biases'] = b
    np.savez(os.path.join(path, 'weights.npz'), **w)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--frames', type=int, default=64)
    ap.add_argument('--points', type=int, default=20000)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--runs', nargs='+', default=['pointgnn_b200.run:1', 'pointgnn_b200.run:8'])
    ap.add_argument('--processes', type=int, nargs='+', default=[1], help='run.py --processes counts to alternate')
    ap.add_argument('--out', default='', help='also write the JSON lines to this file')
    args = ap.parse_args()
    from oracle import kitti as ok
    tmp = tempfile.mkdtemp(prefix='prof_run_')
    lines = []
    try:
        root = os.path.join(tmp, 'kitti')
        ok.write_synthetic_kitti(root, list(range(1000, 1000 + args.frames)), args.points)
        ckpt = os.path.join(tmp, 'ckpt')
        make_checkpoint(ckpt)
        runs = [(spec.rsplit(':', 1)[0], int(spec.rsplit(':', 1)[1]), processes)
                for spec in args.runs for processes in args.processes]

        def once(module, batch_size, processes):
            argv = [ckpt, '--test', '--dataset_root_dir', root, '--output_dir', os.path.join(tmp, 'out')]
            if batch_size != 1:
                argv += ['--batch_size', str(batch_size)]
            if processes != 1:
                argv += ['--processes', str(processes)]
            t0 = time.time()
            times = importlib.import_module(module).main(argv)
            return times, time.time() - t0

        for run in runs:
            once(*run)
        import torch
        conditions = gpu_conditions()
        devices = torch.cuda.device_count()
        for rep in range(args.repeats):
            for module, batch_size, processes in runs:
                times, wall = once(module, batch_size, processes)
                line = {'module': module, 'batch_size': batch_size, 'processes': processes, 'repeat': rep,
                        'frames': args.frames, 'points': args.points, 'frames_per_s': args.frames / times['total'],
                        'stage_ms_per_frame': {k: 1e3 * v / args.frames for k, v in times.items()},
                        'main_wall_s': wall, 'gpu': conditions, 'cuda_devices': devices}
                lines.append(line)
                print(json.dumps(line), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(''.join(json.dumps(line) + '\n' for line in lines))


if __name__ == '__main__':
    main()

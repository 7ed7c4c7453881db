"""Time the beam downsampling (pg_beam_downsample: exact 1-D k-means + bands + compaction) on seeded full-size frames.

    python tools/prof_beam_downsample.py [--points 120000] [--batches 1,16] [--clusters 64] [--reps 5]
        [--sklearn_frames 2] [--out prof_beam_downsample.json]

GPU: CUDA events around whole calls of ``beam_downsample_batch`` (one host round trip each) on batches of
seeded 120 000-point velodyne frames (oracle.beam_downsample.velodyne_frame), after a warm-up call per batch
size; reported per call and per frame, median and spread over the repetitions.  Host: the reference's clustering
step, scikit-learn ``KMeans(n_clusters, n_init=10)`` on one frame's cosines, timed with a wall clock per frame.
The card's name and power limit are read in the same run and printed beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--points', type=int, default=120000)
    ap.add_argument('--batches', type=str, default='1,16')
    ap.add_argument('--clusters', type=int, default=64)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--sklearn_frames', type=int, default=2)
    ap.add_argument('--out', type=str, default='')
    args = ap.parse_args()
    import torch
    from oracle import beam_downsample as obd
    from pointgnn_b200.dataset.kitti_dataset import beam_downsample_batch
    assert torch.cuda.is_available(), 'needs a GPU'
    batches = [int(b) for b in args.batches.split(',')]
    frames = [obd.velodyne_frame(100 + i, args.points) for i in range(max(batches))]
    result = {'card': card(), 'points_per_frame': args.points, 'clusters': args.clusters, 'gpu': {}}
    print('card:', result['card'])
    for bs in batches:
        fp = torch.tensor(np.concatenate([[0], np.cumsum([len(v) for v in frames[:bs]])]), dtype=torch.int32).cuda()
        velo = torch.from_numpy(np.vstack(frames[:bs])).cuda()
        beam_downsample_batch(velo, fp, 2, args.clusters)          # warm-up
        times = []
        for _ in range(args.reps):
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            beam_downsample_batch(velo, fp, 2, args.clusters)
            stop.record()
            stop.synchronize()
            times.append(start.elapsed_time(stop))
        med = float(np.median(times))
        result['gpu'][bs] = {'ms_per_call': med, 'ms_per_frame': med / bs, 'min_ms': min(times), 'max_ms': max(times)}
        print('GPU batch %2d: %.2f ms per call (%.2f-%.2f), %.2f ms per frame' % (bs, med, min(times), max(times),
                                                                               med / bs))
    if args.sklearn_frames > 0:
        from sklearn.cluster import KMeans
        secs = []
        for v in frames[:args.sklearn_frames]:
            cos = obd.cosines(v[:, :3]).reshape(-1, 1)
            t0 = time.time()
            KMeans(n_clusters=args.clusters, n_init=10, random_state=0).fit(cos)
            secs.append(time.time() - t0)
        result['sklearn_s_per_frame'] = float(np.median(secs))
        result['host_cpus'] = os.cpu_count()
        print('host scikit-learn KMeans(n_init=10): %.2f s per frame (%d CPUs)' % (np.median(secs), os.cpu_count()))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()

"""Time the KITTI evaluator twin against the reference evaluator on a seeded KITTI-val-sized tree.

    python tools/prof_eval.py [--frames 3769] [--repeats 5]

Builds a seeded synthetic tree (oracle/kitti_eval.synthetic_tree: car, pedestrian and cyclist labels and results) in
a temporary directory and times, separately: parsing the files on the host; pg_kitti_eval on the device (CUDA events,
after a warm-up call, over --repeats calls; each call ends in its one synchronising read-back); and, when
oracle/_ref/evaluate_object_3d_offline was built, the reference evaluator on the same tree (CPU wall clock, one core).
The outputs of the two are compared in the same run.  Prints one JSON line, with the card and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True, check=True).stdout.strip().split('\n')[0]
    name, power = [x.strip() for x in out.split(',')]
    return name, power


def compare(files, res_dir):
    """-> names of the files whose text differs (similarity files: beyond the half-unit of %f)."""
    bad = []
    for rel, text in files.items():
        path = os.path.join(res_dir, rel)
        if not os.path.isfile(path):
            bad.append(rel)
            continue
        with open(path) as f:
            want = f.read()
        if 'orientation' in rel:
            a, b = text.split(), want.split()
            if len(a) != len(b) or any(x != y and abs(float(x) - float(y)) > 5.01e-7 for x, y in zip(a, b)):
                bad.append(rel)
        elif text != want:
            bad.append(rel)
    return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=3769)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--seed', type=int, default=2024)
    args = ap.parse_args()
    import numpy as np
    import torch
    assert torch.cuda.is_available(), 'prof_eval.py measures the GPU path; there is no CPU fallback'
    from oracle import kitti_eval as ke
    from oracle import kitti_eval_build
    from pointgnn_b200 import _lib
    from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev

    tmp = tempfile.mkdtemp()
    gt_dir, res_dir = os.path.join(tmp, 'label_2'), os.path.join(tmp, 'results')
    ke.write_tree(gt_dir, res_dir, *ke.synthetic_tree(args.seed, args.frames, score_digits=3))

    t0 = time.perf_counter()
    _, groundtruth, detections = ev.load_tree(gt_dir, res_dir)
    parse_s = time.perf_counter() - t0
    num_gt = sum(len(g[0]) for g in groundtruth)
    num_det = sum(len(d[0]) for d in detections)

    compute_aos, evaluated = ev.eval_flags(detections)
    gt_class, gt, gt_ptr = ev._stack(groundtruth, ev.GT_FIELDS)
    det_class, det, det_ptr = ev._stack(detections, ev.DET_FIELDS)
    dev = torch.device('cuda', 0)
    tensors = [torch.from_numpy(a).to(dev) for a in (gt, gt_class, det, det_class)]
    _lib.kitti_eval(*tensors, gt_ptr, det_ptr, compute_aos)              # warm-up
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(args.repeats):
        start.record()
        raw = _lib.kitti_eval(*tensors, gt_ptr, det_ptr, compute_aos)
        stop.record()
        torch.cuda.synchronize()
        times.append(start.elapsed_time(stop) / 1e3)
    t0 = time.perf_counter()
    result = ev.evaluate_frames(groundtruth, detections)
    torch.cuda.synchronize()
    frames_call_s = time.perf_counter() - t0
    assert np.array_equal(result['tp'], raw['tp'])

    line = {'frames': args.frames, 'gt_rows': num_gt, 'detections': num_det, 'host_parse_s': round(parse_s, 4),
            'device_eval_s_median': round(float(np.median(times)), 5), 'device_eval_s_min': round(min(times), 5),
            'device_eval_repeats': args.repeats, 'evaluate_frames_s': round(frames_call_s, 4),
            'thresholds': int(raw['num_thresholds'].sum())}
    binary = kitti_eval_build.binary()
    if binary:
        t0 = time.perf_counter()
        subprocess.run([binary, gt_dir, res_dir], capture_output=True, text=True, check=True)
        line['reference_cpu_s'] = round(time.perf_counter() - t0, 3)
        bad = compare(result['files'], res_dir)
        line['outputs_match_reference'] = not bad
        line['mismatched_files'] = bad
        line['speedup_device_vs_reference'] = round(line['reference_cpu_s'] / float(np.median(times)), 1)
    else:
        line['reference_cpu_s'] = None
    line['gpu'], line['power_limit'] = card()
    print(json.dumps(line))


if __name__ == '__main__':
    main()

"""Score KITTI object-detection result files on the GPU: the twin of the reference's
``kitti_native_evaluation/src/evaluate_object_3d_offline.cpp``.

    python -m pointgnn_b200.kitti_native_evaluation.evaluate_object_3d_offline GT_DIR RESULT_DIR

GT_DIR holds KITTI label files (``NNNNNN.txt``); RESULT_DIR/data/ holds the result files ``run.py`` writes.  For
car, pedestrian and cyclist, and for the image, bird's-eye-view (BEV) and 3D box overlaps, it computes the 41-point
precision / recall curves at the easy, moderate and hard difficulties, and the orientation similarity (AOS, image)
and heading similarity (AHS, BEV and 3D), as the reference evaluator does.  The matching, thresholds and sums run
on the GPU (``pg_kitti_eval``, point-gnn_b200/csrc/pg_eval.cu); this module parses the files and formats the output.

It writes the reference's files, with the same names and contents, into RESULT_DIR:

* ``stats_<cls>_detection.txt`` and ``stats_<cls>_orientation.txt`` (image metric; the second only when no detection
  has ``alpha == -10``), three rows of 41 values: easy, moderate, hard;
* ``stats_<cls>_detection_ground.txt``: the reference opens this file for the BEV metric and opens it again for the
  3D metric, so when a class has 3D results the file holds the 3D rows;
* ``plot/<cls>_{detection_AP, orientation_AOS, detection_BEV_AP, orientation_BEV_AHS, detection_3D_AP,
  orientation_3D_AHS}.txt`` (recall, easy, moderate, hard per line) and a gnuplot script ``.gp`` beside each.

and prints the same lines: ``  done.`` after loading, then ``<name> : easy moderate hard`` AP per curve (the float32
sum of the curve at recall 0, 0.1, ..., 1, over 11, times 100).  The reference also runs gnuplot, ps2pdf and pdfcrop
on the ``.gp`` files; this module does not: run ``gnuplot <name>.gp`` in RESULT_DIR/plot/ to get the EPS plots.

A class is evaluated for a metric only if some detection of it has valid fields for that metric (image:
``x1 >= 0``; BEV: ``t1, t3 != -1000`` and ``w, l > 0``; 3D: also ``t2 != -1000`` and ``h > 0``).

Where the reference is undefined or depends on the order of directory entries, this module does the following:

* frames are evaluated in ascending index order (the reference uses ``readdir`` order; only the AOS / AHS sums'
  last bits can depend on it);
* the index of a result file is the number in the last 10 characters of its name (as there); names shorter than 10
  characters are skipped (as there), and any other name whose last 10 characters are not ``DDDDDD.txt`` raises
  ``ValueError``;
* a record with the wrong number of fields or a malformed number raises ``ValueError`` naming the file and line (the
  reference's ``fscanf`` loop silently re-synchronises); blank lines are skipped;
* a missing ground-truth file raises ``FileNotFoundError``;
* at most 41 score thresholds are used per curve; the reference writes past its 41-entry arrays when there are more.
"""
import os
import re
import sys

import numpy as np

CLASS_NAMES = ['car', 'pedestrian', 'cyclist']
N_SAMPLE_PTS = 41
GT_FIELDS, DET_FIELDS = 14, 15       # numbers after the type in a label / result record
_CODES = {b'car': 0, b'pedestrian': 1, b'cyclist': 2, b'van': 3, b'person_sitting': 4, b'dontcare': 5}
_RESULT_NAME = re.compile(r'[0-9]{6}\.txt')


def class_code(name):
    """The type as pg_kitti_eval's code, compared case-insensitively (ASCII, as strcasecmp)."""
    return _CODES.get(name.encode().lower(), 6)


# ---------------------------------------------------------------------------------------------
# files
# ---------------------------------------------------------------------------------------------
def _read_records(path, num_values, int_column=None):
    names, rows = [], []
    with open(path, encoding='latin-1') as f:
        for lineno, line in enumerate(f, 1):
            fields = line.split()
            if not fields:
                continue
            if len(fields) != num_values + 1:
                raise ValueError('%s:%d: expected %d fields, found %d' % (path, lineno, num_values + 1, len(fields)))
            try:
                values = [float(v) for v in fields[1:]]
                if int_column is not None:
                    values[int_column] = float(int(fields[1 + int_column]))
            except ValueError:
                raise ValueError('%s:%d: malformed number in %r' % (path, lineno, line.rstrip('\n'))) from None
            names.append(fields[0])
            rows.append(values)
    return names, np.asarray(rows, dtype=np.float64).reshape(len(rows), num_values)


def read_groundtruth(path):
    """A KITTI label file (loadGroundtruth) -> (types, [G, 14] float64: truncation, occlusion, alpha, x1, y1, x2, y2,
    h, w, l, t1, t2, t3, ry).  The occlusion must be an integer, as the reference's ``%d``."""
    return _read_records(path, GT_FIELDS, int_column=1)


def read_detections(path):
    """A KITTI result file (loadDetections) -> (types, [D, 15] float64: two unused, alpha, x1, y1, x2, y2, h, w, l,
    t1, t2, t3, ry, score)."""
    return _read_records(path, DET_FIELDS)


def frame_indices(data_dir):
    """getEvalIndices: the frame index of every result file, ascending."""
    indices = []
    for name in os.listdir(data_dir):
        if len(name) < 10:
            continue
        if not _RESULT_NAME.fullmatch(name[-10:]):
            raise ValueError('%s: result file names must end in DDDDDD.txt' % os.path.join(data_dir, name))
        indices.append(int(name[-10:-4]))
    return sorted(indices)


# ---------------------------------------------------------------------------------------------
# evaluation
# ---------------------------------------------------------------------------------------------
def eval_flags(detections):
    """What loadDetections decides while reading: compute_aos, and per class whether the image / BEV / 3D metrics
    are evaluated (:152-167)."""
    compute_aos = True
    flags = np.zeros((3, 3), dtype=bool)          # [metric, class]
    for names, v in detections:
        if len(names) == 0:
            continue
        if np.any(v[:, 2] == -10):
            compute_aos = False
        codes = np.array([class_code(n) for n in names])
        t1, t2, t3, h, w, l = v[:, 10], v[:, 11], v[:, 12], v[:, 7], v[:, 8], v[:, 9]
        ground = (t1 != -1000) & (t3 != -1000) & (w > 0) & (l > 0)
        box3d = ground & (t2 != -1000) & (h > 0)
        for c in range(3):
            mine = codes == c
            flags[0, c] |= bool(np.any(mine & (v[:, 3] >= 0)))
            flags[1, c] |= bool(np.any(mine & ground))
            flags[2, c] |= bool(np.any(mine & box3d))
    return compute_aos, flags


def _stack(frames, width):
    names = [n for f in frames for n in f[0]]
    values = np.concatenate([np.asarray(f[1], np.float64).reshape(-1, width) for f in frames] +
                            [np.zeros((0, width))])
    ptr = np.zeros(len(frames) + 1, np.int64)
    ptr[1:] = np.cumsum([len(f[0]) for f in frames])
    return np.array([class_code(n) for n in names], np.int32), values, ptr


def evaluate_frames(groundtruth, detections):
    """Evaluate per-frame arrays: ``groundtruth[f] = (types, [G_f, 14])`` and ``detections[f] = (types, [D_f, 15])`` as
    read_groundtruth / read_detections return them.  -> dict with

    * ``curves``: output name -> [3, 41] (easy, moderate, hard) and ``ap``: output name -> the three printed AP values,
      both in the reference's output order;
    * ``files``: path relative to RESULT_DIR -> text, ``lines``: the printed lines after ``  done.``;
    * ``precision`` / ``aos`` / ``ahs`` [3, 3, 3, 41], ``tp`` / ``fp`` / ``fn`` [3, 3, 3, 41], ``num_thresholds`` [3, 3, 3]
      (axes metric, class, difficulty, threshold) and ``compute_aos`` / ``evaluated`` [metric, class]."""
    if len(groundtruth) != len(detections):
        raise ValueError('%d ground-truth frames, %d detection frames' % (len(groundtruth), len(detections)))
    compute_aos, evaluated = eval_flags(detections)
    if evaluated.any():
        import torch
        from pointgnn_b200 import _lib
        gt_class, gt, gt_ptr = _stack(groundtruth, GT_FIELDS)
        det_class, det, det_ptr = _stack(detections, DET_FIELDS)
        dev = torch.device('cuda', torch.cuda.current_device())
        raw = _lib.kitti_eval(torch.from_numpy(gt).to(dev), torch.from_numpy(gt_class).to(dev),
                              torch.from_numpy(det).to(dev), torch.from_numpy(det_class).to(dev), gt_ptr, det_ptr,
                              compute_aos)
    else:   # no class is evaluated under any metric: nothing to compute, nothing written
        raw = {k: np.zeros((3, 3, 3, 41)) for k in ('precision', 'aos', 'ahs', 'tp', 'fp', 'fn')}
        raw['num_thresholds'] = np.zeros((3, 3, 3), np.int32)
    return report(raw, compute_aos, evaluated)


def _f(v):
    # printf("%f"): every NaN here comes from 0 / 0, which x86 produces with the sign bit set
    return '-nan' if v != v else '%f' % v


def printed_ap(curve):
    """printAp / saveAndPlotPlots: float32 sum of entries 0, 4, ..., 40 of each difficulty, / 11 * 100."""
    out = []
    for v in curve:
        s = np.float32(0)
        for i in range(0, len(v), 4):
            s = np.float32(np.float64(s) + v[i])
        out.append(float(s / np.float32(11) * np.float32(100)))
    return tuple(out)


def _gnuplot(name, cls, is_aos):
    # the second (eps) version saveAndPlotPlots writes, which is the file's final content
    return ''.join([
        'set term postscript eps enhanced color font "Helvetica" 20\n',
        'set output "%s.eps"\n' % name,
        'set size ratio 0.7\n', 'set xrange [0:1]\n', 'set yrange [0:1]\n', 'set xlabel "Recall"\n',
        'set ylabel "Orientation Similarity"\n' if is_aos else 'set ylabel "Precision"\n',
        'set title "%s"\n' % (cls[:1].upper() + cls[1:]),
        'plot ',
        '"%s.txt" using 1:2 title \'Easy\' with lines ls 1 lw 5,' % name,
        '"%s.txt" using 1:3 title \'Moderate\' with lines ls 2 lw 5,' % name,
        '"%s.txt" using 1:4 title \'Hard\' with lines ls 3 lw 5' % name])


def report(raw, compute_aos, evaluated):
    """The reference's output files and printed lines from the [metric, class, difficulty, 41] curves."""
    out = dict(raw)
    out.update(compute_aos=compute_aos, evaluated=evaluated, files={}, lines=[], curves={}, ap={})

    def stats(curve):
        return ''.join(''.join(_f(x) + ' ' for x in row) + '\n' for row in curve)

    def plot(name, cls, curve, is_aos):
        out['files']['plot/%s.txt' % name] = ''.join(
            '%f %s %s %s\n' % (i / (N_SAMPLE_PTS - 1.0), _f(curve[0][i]), _f(curve[1][i]), _f(curve[2][i]))
            for i in range(N_SAMPLE_PTS))
        ap = printed_ap(curve)
        out['lines'].append('%s : %s %s %s' % ((name,) + tuple(_f(a) for a in ap)))
        out['files']['plot/%s.gp' % name] = _gnuplot(name, cls, is_aos)
        out['curves'][name] = np.array(curve)
        out['ap'][name] = ap

    prec, aos, ahs = raw['precision'], raw['aos'], raw['ahs']
    for c, cls in enumerate(CLASS_NAMES):
        if evaluated[0, c]:
            out['files']['stats_%s_detection.txt' % cls] = stats(prec[0, c])
            if compute_aos:
                out['files']['stats_%s_orientation.txt' % cls] = stats(aos[0, c])
            plot(cls + '_detection_AP', cls, prec[0, c], False)
            if compute_aos:
                plot(cls + '_orientation_AOS', cls, aos[0, c], True)
    for m, tag in ((1, 'BEV'), (2, '3D')):
        for c, cls in enumerate(CLASS_NAMES):
            if evaluated[m, c]:
                out['files']['stats_%s_detection_ground.txt' % cls] = stats(prec[m, c])
                plot('%s_detection_%s_AP' % (cls, tag), cls, prec[m, c], False)
                plot('%s_orientation_%s_AHS' % (cls, tag), cls, ahs[m, c], True)
    return out


def load_tree(gt_dir, result_dir):
    """The frames of a result tree, in ascending index order -> (indices, groundtruth, detections)."""
    data_dir = os.path.join(result_dir, 'data')
    indices = frame_indices(data_dir)
    groundtruth, detections = [], []
    for idx in indices:
        name = '%06d.txt' % idx
        gt_path = os.path.join(gt_dir, name)
        if not os.path.isfile(gt_path):
            raise FileNotFoundError("Couldn't read: %s of ground truth" % gt_path)
        groundtruth.append(read_groundtruth(gt_path))
        detections.append(read_detections(os.path.join(data_dir, name)))
    return indices, groundtruth, detections


def write_report(result_dir, result):
    """Write result['files'] under result_dir (plot/ is created even when nothing is evaluated, as there)."""
    os.makedirs(os.path.join(result_dir, 'plot'), exist_ok=True)
    for rel, text in result['files'].items():
        with open(os.path.join(result_dir, rel), 'w') as f:
            f.write(text)


def evaluate(gt_dir, result_dir):
    """evaluate_object_3d_offline GT_DIR RESULT_DIR: parse, evaluate on the GPU, write the files, print the lines.
    Returns what evaluate_frames returns."""
    _, groundtruth, detections = load_tree(gt_dir, result_dir)
    print('  done.')
    result = evaluate_frames(groundtruth, detections)
    write_report(result_dir, result)
    for line in result['lines']:
        print(line)
    return result


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    if len(argv) != 2:
        print('Usage: ./eval_detection_3d_offline gt_dir result_dir')
        return 1
    evaluate(argv[0], argv[1])
    return 0


if __name__ == '__main__':
    sys.exit(main())

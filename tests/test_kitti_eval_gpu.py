"""GPU tests of the KITTI evaluator twin (pg_kitti_eval, pointgnn_b200.kitti_native_evaluation): the reference
evaluator's goldens, exact counts against the NumPy restatement on larger seeded trees, run-to-run identity, the
array and file entry points, and a result tree written by the run.py twin."""
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN
from test_kitti_eval_cpu import TREES, expected_lines, load_golden_tree

pytestmark = pytest.mark.gpu


def _numbers_close(got, want, tol):
    """Whitespace-separated tokens: '-nan' and non-numbers equal, numbers within tol."""
    a, b = got.split(), want.split()
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        if x == y:
            continue
        try:
            if not abs(float(x) - float(y)) <= tol:
                return False
        except ValueError:
            return False
    return True


def _ev():
    from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev
    return ev


@pytest.mark.parametrize('tree', TREES)
def test_gpu_reproduces_reference_goldens(tree, tmp_path, capsys):
    gt_dir, res_dir, g = load_golden_tree(tree, tmp_path)
    _ev().evaluate(gt_dir, res_dir)
    printed = capsys.readouterr().out
    produced = set()
    for d, _, files in os.walk(res_dir):
        for fname in files:
            rel = os.path.relpath(os.path.join(d, fname), res_dir)
            if not rel.startswith('data' + os.sep):
                produced.add(rel)
    assert produced == set(g['outputs'])
    for rel, want in g['outputs'].items():
        with open(os.path.join(res_dir, rel)) as f:
            got = f.read()
        similarity = 'orientation' in rel
        if not similarity:
            assert got == want, rel                     # precision curves and gnuplot scripts: as text
        else:                                           # AOS / AHS: within the half-unit of %f
            assert _numbers_close(got, want, 5.01e-7), rel
    got_lines, want_lines = printed.split('\n'), g['stdout'].split('\n')
    assert len(got_lines) == len(want_lines)
    for a, b in zip(got_lines, want_lines):
        if 'orientation' in b:     # float32 sums of the similarity curves: one float32 step of slack
            name_a, _, va = a.partition(' : ')
            name_b, _, vb = b.partition(' : ')
            assert name_a == name_b and _numbers_close(va, vb, 2e-6), (a, b)
        else:
            assert a == b


def _big_tree(seed, frames=500):
    from oracle import kitti_eval as ke
    return ke.synthetic_tree(seed, frames, big_frames=tuple(range(10, frames, 50)), score_digits=3)


def _frames(tmp_path, texts):
    from oracle import kitti_eval as ke
    gt_dir, res_dir = str(tmp_path / 'gt'), str(tmp_path / 'res')
    ke.write_tree(gt_dir, res_dir, *texts)
    return gt_dir, res_dir


def _assert_same_counts(got, want):
    for k in ('num_thresholds', 'tp', 'fp', 'fn', 'precision'):
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k]), equal_nan=True), k
    for k in ('aos', 'ahs'):
        a, b = np.asarray(got[k]), np.asarray(want[k])
        assert np.array_equal(np.isnan(a), np.isnan(b)), k
        ok = ~np.isnan(a)
        assert np.all(np.abs(a[ok] - b[ok]) <= 1e-12 * np.maximum(np.abs(b[ok]), 1e-300)), k


@pytest.mark.parametrize('seed', [51, 52])
def test_counts_equal_restatement_on_large_trees(seed, tmp_path):
    from oracle import kitti_eval as ke
    ev = _ev()
    gt_dir, res_dir = _frames(tmp_path, _big_tree(seed))
    _, groundtruth, detections = ev.load_tree(gt_dir, res_dir)
    assert len(groundtruth) >= 500 and max(len(d[0]) for d in detections) >= 200
    got = ev.evaluate_frames(groundtruth, detections)
    want = ke.evaluate_arrays(groundtruth, detections)
    assert got['num_thresholds'].sum() > 100
    _assert_same_counts(got, want)


def test_matches_compiled_reference_on_fresh_tree(tmp_path, capsys):
    from oracle import kitti_eval_build
    binary = kitti_eval_build.binary()
    if binary is None:
        pytest.skip('oracle/_ref/evaluate_object_3d_offline was not built (no reference tree)')
    from oracle import kitti_eval as ke
    texts = ke.synthetic_tree(77, 120, big_frames=(30,))
    gt_a, res_a = _frames(tmp_path / 'a', texts)
    gt_b, res_b = _frames(tmp_path / 'b', texts)
    out = subprocess.run([binary, gt_b, res_b], capture_output=True, text=True, check=True).stdout
    r = _ev().evaluate(gt_a, res_a)
    assert capsys.readouterr().out.split('\n')[0] == '  done.'
    for rel, text in r['files'].items():
        with open(os.path.join(res_b, rel)) as f:
            want = f.read()
        if 'orientation' in rel:
            assert _numbers_close(text, want, 5.01e-7), rel
        else:
            assert text == want, rel
    assert len(r['lines']) == len(expected_lines({'stdout': out}))


def test_two_calls_give_identical_files(tmp_path):
    ev = _ev()
    texts = _big_tree(61, 200)
    outs = []
    for k in range(2):
        gt_dir, res_dir = _frames(tmp_path / str(k), texts)
        ev.evaluate(gt_dir, res_dir)
        files = {}
        for d, _, names in os.walk(res_dir):
            for n in names:
                with open(os.path.join(d, n), 'rb') as f:
                    files[os.path.relpath(os.path.join(d, n), res_dir)] = f.read()
        outs.append(files)
    assert outs[0] == outs[1]


def test_evaluate_frames_equals_evaluate(tmp_path):
    ev = _ev()
    gt_dir, res_dir, _ = load_golden_tree('mixed', tmp_path)
    a = ev.evaluate(gt_dir, res_dir)
    _, groundtruth, detections = ev.load_tree(gt_dir, res_dir)
    b = ev.evaluate_frames(groundtruth, detections)
    assert a['files'] == b['files'] and a['lines'] == b['lines'] and list(a['ap']) == list(b['ap'])
    for k in ('precision', 'aos', 'ahs', 'tp', 'fp', 'fn', 'num_thresholds'):
        assert np.array_equal(a[k], b[k], equal_nan=True), k


def test_cli(tmp_path):
    import sys
    gt_dir, res_dir, g = load_golden_tree('no_aos_no_cyclist', tmp_path)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, '-m', 'pointgnn_b200.kitti_native_evaluation.evaluate_object_3d_offline',
                          gt_dir, res_dir], capture_output=True, text=True, cwd=root, check=True).stdout
    assert out.split('\n')[0] == '  done.' and len(out.split('\n')) == len(g['stdout'].split('\n'))
    with open(os.path.join(res_dir, 'stats_car_detection.txt')) as f:
        assert f.read() == g['outputs']['stats_car_detection.txt']


def test_run_twin_result_tree(tmp_path):
    """A result tree written by pointgnn_b200.run scores the same on the GPU and in the restatement."""
    from oracle import kitti as ok
    from oracle import kitti_eval as ke
    from pointgnn_b200 import run as twin
    ev = _ev()
    root = str(tmp_path / 'kitti')
    names = ok.write_synthetic_kitti(root, [41, 42, 43], 6000)
    ckpt = tmp_path / 'ckpt'
    ckpt.mkdir()
    shutil.copy(os.path.join(GOLDEN, 'config_car_auto_T3_train.json'), str(ckpt / 'config'))
    # as tests/test_kitti_gpu.py: the real weights with the object-class logit biases raised, so that the model fires
    w = dict(np.load(os.path.join(GOLDEN, 'weights_car_auto_T3_train.npz')))
    b = w['output/predictor/cls/fully_connected_1/biases'].copy()
    b[1:-1] += 7.0
    w['output/predictor/cls/fully_connected_1/biases'] = b
    np.savez(str(ckpt / 'weights.npz'), **w)
    out_dir = str(tmp_path / 'out')
    twin.main([str(ckpt), '--test', '--dataset_root_dir', root, '--output_dir', out_dir])
    # labels: every third detection jittered into a ground-truth box, plus one DontCare region per frame
    rng = np.random.default_rng(5)
    gt_dir = str(tmp_path / 'label_2')
    os.makedirs(gt_dir)
    for name in names:
        _, dets = ev.read_detections(os.path.join(out_dir, 'data', name + '.txt'))
        rows = []
        for d in dets[::3]:
            x1, y1, x2, y2 = d[3:7] + rng.normal(0, 2, 4)
            h, w_, l, t1, t2, t3, ry = d[7:14] + rng.normal(0, 0.1, 7)
            rows.append('Car %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f' % (
                rng.choice([0.0, 0.2, 0.4]), rng.integers(0, 3), d[2], x1, y1, x1 + max(x2 - x1, 1), y1 + max(y2 - y1, 1),
                h, w_, l, t1, t2, t3, ry))
        rows.append('DontCare -1 -1 -10 500 150 600 200 -1 -1 -1 -1000 -1000 -1000 -10')
        with open(os.path.join(gt_dir, name + '.txt'), 'w') as f:
            f.write('\n'.join(rows) + '\n')
    _, groundtruth, detections = ev.load_tree(gt_dir, out_dir)
    assert sum(len(d[0]) for d in detections) > 0
    got = ev.evaluate_frames(groundtruth, detections)
    want = ke.evaluate_frames(groundtruth, detections)
    _assert_same_counts(got, want)
    assert got['files'].keys() == want['files'].keys()
    assert [l for l in got['lines'] if 'orientation' not in l] == [l for l in want['lines'] if 'orientation' not in l]

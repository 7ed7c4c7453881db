"""CPU tests of the KITTI evaluator twin: the NumPy restatement (oracle/kitti_eval.py) and the compiled reference
evaluator reproduce the committed goldens; the result-file parser reads what our writer emits and rejects what it
cannot read."""
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN

TREES = ['mixed', 'no_aos_no_cyclist']


def load_golden_tree(name, tmp_path):
    """Write a golden tree under tmp_path -> (gt_dir, result_dir, golden dict)."""
    with open(os.path.join(GOLDEN, 'kitti_eval_%s.json' % name)) as f:
        g = json.load(f)
    gt_dir, res_dir = str(tmp_path / 'label_2'), str(tmp_path / 'results')
    os.makedirs(gt_dir)
    os.makedirs(os.path.join(res_dir, 'data'))
    for sub, d in (('label_2', gt_dir), ('data', os.path.join(res_dir, 'data'))):
        for fname, text in g[sub].items():
            with open(os.path.join(d, fname), 'w') as f:
                f.write(text)
    return gt_dir, res_dir, g


def expected_lines(g):
    lines = g['stdout'].split('\n')
    assert lines[0] == '  done.' and lines[-1] == ''
    return lines[1:-1]


@pytest.mark.parametrize('tree', TREES)
def test_restatement_reproduces_reference_goldens(tree, tmp_path):
    from oracle import kitti_eval as ke
    gt_dir, res_dir, g = load_golden_tree(tree, tmp_path)
    r = ke.evaluate_tree(gt_dir, res_dir)
    assert sorted(r['files']) == sorted(g['outputs'])
    for rel, text in g['outputs'].items():
        assert r['files'][rel] == text, rel
    assert r['lines'] == expected_lines(g)


@pytest.mark.parametrize('tree', TREES)
def test_compiled_reference_reproduces_goldens(tree, tmp_path):
    from oracle import kitti_eval_build
    binary = kitti_eval_build.binary()
    if binary is None:
        pytest.skip('oracle/_ref/evaluate_object_3d_offline was not built (no reference tree)')
    gt_dir, res_dir, g = load_golden_tree(tree, tmp_path)
    out = subprocess.run([binary, gt_dir, res_dir], capture_output=True, text=True, check=True).stdout
    assert out == g['stdout']
    for rel, text in g['outputs'].items():
        with open(os.path.join(res_dir, rel)) as f:
            assert f.read() == text, rel


def test_goldens_cover_the_cases():
    from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev
    with open(os.path.join(GOLDEN, 'kitti_eval_mixed.json')) as f:
        g = json.load(f)
    types = {line.split()[0] for t in g['label_2'].values() for line in t.split('\n') if line.strip()}
    assert {'Car', 'car', 'Van', 'Pedestrian', 'Person_sitting', 'Cyclist', 'DontCare', 'Misc'} <= types
    assert any(t == '' for t in g['label_2'].values()), 'an empty label file'
    assert any(t.strip() == '' for t in g['data'].values()), 'an empty result file'
    dets = [line.split() for t in g['data'].values() for line in t.split('\n') if line.strip()]
    assert any(float(d[11]) == -1000 for d in dets)
    assert max(len(t.split('\n')) for t in g['data'].values()) > 200, 'a frame with > 200 detections'
    scores = [d[15] for d in dets]
    assert len(set(scores)) < len(scores), 'tied scores'
    assert any(float(d[7]) - float(d[5]) != int(float(d[7]) - float(d[5])) for d in dets)
    with open(os.path.join(GOLDEN, 'kitti_eval_no_aos_no_cyclist.json')) as f:
        g2 = json.load(f)
    assert not any(n.startswith('stats_cyclist') for n in g2['outputs'])
    assert not any('orientation_AOS' in n for n in g2['outputs'])
    assert ev.class_code('cYcList') == 2 and ev.class_code('DONTCARE') == 5 and ev.class_code('Truck') == 6


def test_parser_reads_our_writer(tmp_path):
    from pointgnn_b200 import run
    from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev
    labels = [('Car', -1, -1, 0, np.float32(10.5), np.float32(20.25), np.float32(100.0), np.float32(80.0),
               np.float32(1.5), np.float32(1.6), np.float32(3.9), np.float32(1.0), np.float32(1.7), np.float32(20.0),
               np.float32(0.3), np.float32(0.87654321))]
    path = str(tmp_path / 'data' / '000000.txt')
    run.write_kitti_file(path, labels)
    names, v = ev.read_detections(path)
    assert names == ['Car'] and v.shape == (1, 15)
    assert np.array_equal(v[0], np.array([float(str(x)) for x in labels[0][1:]]))
    run.write_kitti_file(path, [])
    names, v = ev.read_detections(path)
    assert names == [] and v.shape == (0, 15)
    open(str(tmp_path / 'empty.txt'), 'w').close()
    names, v = ev.read_groundtruth(str(tmp_path / 'empty.txt'))
    assert names == [] and v.shape == (0, 14)


def test_parser_errors(tmp_path):
    from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev
    p = tmp_path / 'x.txt'
    p.write_text('Car 0 0 0 1 2 3 4 1 1 1 0 0 0 0\n\nCar 0 0 0 1 2 3\n')
    with pytest.raises(ValueError, match='x.txt:3'):
        ev.read_groundtruth(str(p))
    p.write_text('Car 0 0.5 0 1 2 3 4 1 1 1 0 0 0 0\n')        # occlusion is an integer (%d)
    with pytest.raises(ValueError, match='x.txt:1'):
        ev.read_groundtruth(str(p))
    p.write_text('Car -1 -1 0 1 2 3 4 1 1 1 0 0 0 0 abc\n')
    with pytest.raises(ValueError, match='malformed'):
        ev.read_detections(str(p))
    data = tmp_path / 'res' / 'data'
    data.mkdir(parents=True)
    (data / '000001.txt').write_text('\n')
    (data / 'a.txt').write_text('\n')                            # shorter than 10 characters: skipped, as there
    assert ev.frame_indices(str(data)) == [1]
    (data / 'frame_00001.txt').write_text('\n')
    with pytest.raises(ValueError):
        ev.frame_indices(str(data))
    os.remove(str(data / 'frame_00001.txt'))
    (tmp_path / 'gt').mkdir()
    with pytest.raises(FileNotFoundError):
        ev.evaluate(str(tmp_path / 'gt'), str(tmp_path / 'res'))


def test_frames_in_ascending_index_order(tmp_path):
    from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev
    data = tmp_path / 'data'
    data.mkdir()
    for i in (12, 3, 100, 7):
        (data / ('%06d.txt' % i)).write_text('\n')
    (data / 'run_000005.txt').write_text('\n')
    assert ev.frame_indices(str(data)) == [3, 5, 7, 12, 100]


def test_printed_ap_is_a_float32_sum():
    from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev
    curve = np.full((3, 41), 0.1)
    s = np.float32(0)
    for _ in range(11):
        s = np.float32(np.float64(s) + 0.1)
    assert ev.printed_ap(curve)[0] == float(s / np.float32(11) * np.float32(100))
    assert ev._f(float('nan')) == '-nan' and ev._f(0.5) == '0.500000'

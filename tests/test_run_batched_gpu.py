"""run.py --batch_size N on a synthetic KITTI-format tree: the files do not depend on N, and they match the CPU oracle
pipeline frame by frame.

Five frames: four oracle/synth.py scenes and one cloud of points a couple of metres in front of the camera, whose
boxes all fail the truncation filter, so that its file holds no row.  --batch_size 3 splits them 3 + 2.  Every stage
is row- or frame-independent, so the files of --batch_size 3 and 1 must be byte-identical.  Input features 'i' take
the image size from the PNG header; an 'irgb' copy of the config decodes the images for their colours."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import cpu_reference, kitti as ok, postprocess as pp
from oracle import graph as ograph

pytestmark = pytest.mark.gpu
CFG = 'car_auto_T3_train'
EMPTY = 2          # the frame without rows
TIMERS = {'fetch input', 'gen graph', 'gnn inference', 'decode box', 'nms', 'total'}
FIRST_LAYER = 'layer1/extract_vertex_features/fully_connected/weights'


def _tree(root):
    names = ok.write_synthetic_kitti(root, [41, 42, 0, 43, 44], 6000)
    calib = ok.parse_calib(os.path.join(root, 'calib/testing/calib', names[EMPTY] + '.txt'))
    rng = np.random.default_rng(0)
    cam = np.c_[rng.uniform(-1, 1, 400), rng.uniform(0, 1.5, 400), rng.uniform(1.5, 3, 400)]
    velo = np.matmul(np.hstack([cam, np.ones([400, 1])]), np.transpose(calib['cam_to_velo']))[:, :3]
    data = np.hstack([velo, rng.uniform(0, 1, (400, 1))]).astype(np.float32)
    data.tofile(os.path.join(root, 'velodyne/testing/velodyne', names[EMPTY] + '.bin'))
    return names


def _checkpoint(path, input_features):
    """The end-to-end test's checkpoint: the real car weights with the object-class logit biases raised by 7.  For
    'irgb' the first layer gets three seeded rows for r, g, b after the intensity row."""
    os.makedirs(path)
    with open(os.path.join(GOLDEN, 'config_%s.json' % CFG)) as f:
        config = json.load(f)
    config['input_features'] = input_features
    with open(os.path.join(path, 'config'), 'w') as f:
        json.dump(config, f)
    w = dict(np.load(os.path.join(GOLDEN, 'weights_%s.npz' % CFG)))
    b = w['output/predictor/cls/fully_connected_1/biases'].copy()
    b[1:-1] += 7.0
    w['output/predictor/cls/fully_connected_1/biases'] = b
    if input_features == 'irgb':
        w0 = w[FIRST_LAYER]
        rgb = (np.random.default_rng(1).standard_normal((3, w0.shape[1])) * 0.05).astype(np.float32)
        w[FIRST_LAYER] = np.concatenate([w0[:1], rgb, w0[1:]])
    np.savez(os.path.join(path, 'weights.npz'), **w)
    return config, w


def _oracle_text(root, name, config, weights, rgb):
    velo = np.fromfile(os.path.join(root, 'velodyne/testing/velodyne', name + '.bin'), dtype=np.float32).reshape(-1, 4)
    calib = ok.parse_calib(os.path.join(root, 'calib/testing/calib', name + '.txt'))
    image = None
    if rgb:
        import cv2
        image = cv2.imread(os.path.join(root, 'image/testing/image_2', name + '.png'))
    xyz, attr = ok.cam_points_in_image(velo, calib, 1242, 375, image)
    coords, kp, edges = ograph.gen_multi_level_local_graph_v3(xyz, **config['runtime_graph_gen_kwargs'])
    _, boxes, probs = cpu_reference.predict(weights, config['model_kwargs']['layer_configs'], config['num_classes'], 7,
                                            attr, coords, kp, edges)
    last = coords[config['model_kwargs']['layer_configs'][-1]['graph_level'] + 1]
    dec = pp.decode_boxes(boxes, last, pp.LABEL_MAPS[config['label_method']])
    lab, bx, sc, idx = pp.select_candidates(probs, dec, config['num_classes'])
    want = []
    if len(lab):
        k_lab, k_box, k_sc, _ = pp.nms_boxes_3d_uncertainty(lab, bx, sc, config['nms_overlapped_thres'])
        want = ok.kitti_labels(k_lab, k_box, k_sc, last[idx // config['num_classes']], calib, config['label_method'])
    return ok.format_kitti(want)


@pytest.mark.parametrize('input_features', ['i', 'irgb'])
def test_batched_run_matches_single_frame_run_and_oracle(tmp_path, input_features):
    from pointgnn_b200 import run
    root = str(tmp_path / 'kitti')
    names = _tree(root)
    ckpt = str(tmp_path / 'ckpt')
    config, weights = _checkpoint(ckpt, input_features)
    files = {}
    for batch_size in (3, 1):
        out_dir = str(tmp_path / ('out%d' % batch_size))
        times = run.main([ckpt, '--test', '--dataset_root_dir', root, '--output_dir', out_dir,
                          '--batch_size', str(batch_size)])
        assert set(times) == TIMERS
        files[batch_size] = {}
        for name in names:
            with open(os.path.join(out_dir, 'data', name + '.txt'), 'rb') as f:
                files[batch_size][name] = f.read()
    for name in names:
        assert files[3][name] == files[1][name], name
    assert files[3][names[EMPTY]] == b'\n'
    total_rows = 0
    for name in names:
        got = ok.parse_kitti_text(files[3][name].decode())
        want = ok.parse_kitti_text(_oracle_text(root, name, config, weights, input_features == 'irgb'))
        assert len(got) == len(want), (name, len(got), len(want))
        for (n1, v1), (n2, v2) in zip(got, want):
            assert n1 == n2
            assert np.allclose(v1, v2, rtol=2e-3, atol=2e-3), (name, v1, v2)
        total_rows += len(got)
    assert total_rows > 0, 'the synthetic frames produced no row at all: the test would be vacuous'

"""pg_beam_downsample (dataset.kitti_dataset.beam_downsample_batch and the point_cloud_downsample CLI) on the GPU:
the reference script's bytes given its own centres, the exact 1-D k-means against the NumPy oracle and against
scikit-learn's fits, batch / single-frame and run-to-run identity, the short-frame error, and run.py on the
downsampled tree."""
import hashlib
import os
import shutil

import numpy as np
import pytest
import torch

from conftest import GOLDEN as GOLDEN_DIR
from oracle import beam_downsample as obd
from oracle import kitti as ok

pytestmark = pytest.mark.gpu
GOLDEN = np.load(os.path.join(GOLDEN_DIR, 'beam_downsample.npz'))


def _dev(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def _batch(frames, k, rate=2, centers=None):
    from pointgnn_b200.dataset.kitti_dataset import beam_downsample_batch
    fp = np.concatenate([[0], np.cumsum([len(v) for v in frames])]).astype(np.int32)
    velo = np.vstack(frames).astype(np.float32) if frames else np.zeros((0, 4), np.float32)
    res = beam_downsample_batch(_dev(velo), _dev(fp), rate, k, None if centers is None else _dev(centers, np.float64))
    return {key: val.cpu().numpy() for key, val in res.items()}


def _frames_of(res):
    fp = res['frame_ptr']
    return [res['velo'][fp[f]:fp[f + 1]] for f in range(len(fp) - 1)]


def test_reference_bytes_with_sklearn_centres():
    n = len(GOLDEN['names'])
    frames = [GOLDEN['velo_%d' % i] for i in range(n)]
    res = _batch(frames, int(GOLDEN['num_clusters']), int(GOLDEN['downsample_rate']), GOLDEN['sk_centers'])
    for i, out in enumerate(_frames_of(res)):
        assert out.tobytes() == GOLDEN['bin_%d' % i].tobytes(), i
    from pointgnn_b200.dataset.kitti_dataset import beam_downsample_batch
    out, centers, inertia = beam_downsample_batch(frames[0], None, 2, 64, GOLDEN['sk_centers'][0])
    assert out.tobytes() == GOLDEN['bin_0'].tobytes() and inertia is None
    assert np.array_equal(centers, np.sort(GOLDEN['sk_centers'][0]))


def _special_frames():
    """(name, [M,4] float32 rows, k)"""
    out = []
    for n, k, seed in ((200, 2, 1), (1000, 16, 2), (3000, 33, 3), (5000, 64, 4), (20000, 64, 5), (20000, 7, 6)):
        out.append(('synthetic %d k%d' % (n, k), obd.velodyne_frame(seed, n, full_360=False), k))
    base = obd.velodyne_frame(7, 2000, full_360=False)
    out.append(('duplicated cosines', np.repeat(base[:500], 4, axis=0)[np.random.default_rng(0).permutation(2000)], 24))
    out.append(('fewer distinct values than clusters', np.repeat(base[:10], 30, axis=0), 16))
    zero = base.copy()
    zero[[5, 900]] = [0.0, 0.0, 0.0, 0.5]
    out.append(('zero-norm points', zero, 32))
    out.append(('exactly k points', base[:64], 64))
    return out


@pytest.mark.parametrize('case', range(10))
def test_exact_kmeans_matches_oracle(case):
    name, velo, k = _special_frames()[case]
    res = _batch([velo], k)
    want = obd.exact_kmeans_1d(obd.cosines(velo[:, :3]), k)
    got_i, want_i = float(res['inertia'][0]), want['inertia']
    assert abs(got_i - want_i) <= 1e-12 * want_i, (name, got_i, want_i)
    assert np.abs(res['centers'][0] - want['centers']).max() <= 1e-12, name
    if want['near_ties'] == 0:
        assert np.array_equal(res['group_sizes'][0], want['sizes']), name
    assert int(res['group_sizes'][0].sum()) == int(np.isfinite(obd.cosines(velo[:, :3])).sum())
    mask = obd.band_mask(obd.cosines(velo[:, :3]), res['centers'][0], 2)
    assert res['velo'].tobytes() == velo[mask].tobytes(), name
    if name == 'zero-norm points':
        assert not (res['velo'][:, :3] == 0).all(axis=1).any()
    if name == 'fewer distinct values than clusters':
        assert got_i == 0.0 and len(np.unique(res['centers'][0])) == 10


def test_full_size_frames_not_above_sklearn():
    frames = []
    for seed, sha in zip(GOLDEN['full_seeds'], GOLDEN['full_sha256']):
        velo = obd.velodyne_frame(int(seed), int(GOLDEN['full_num_points']))
        assert hashlib.sha256(velo.tobytes()).hexdigest() == str(sha), 'the synthetic frame is not the recorded one'
        frames.append(velo)
    res = _batch(frames, 64)
    for f in range(len(frames)):
        assert res['inertia'][f] <= GOLDEN['full_sk_inertia'][f] * (1 + 1e-12), (res['inertia'][f],
                                                                                 GOLDEN['full_sk_inertia'][f])


def test_batch_equals_single_frames_and_is_repeatable():
    frames = [obd.velodyne_frame(s, n, full_360=False) for s, n in ((11, 3000), (12, 500), (13, 8000))]
    frames.insert(1, np.zeros((0, 4), np.float32))
    frames.append(np.repeat(frames[0][:7], 5, axis=0))     # 7 distinct values, 16 clusters
    a, b = _batch(frames, 16, 3), _batch(frames, 16, 3)
    for key in a:
        assert a[key].tobytes() == b[key].tobytes(), key
    assert np.isnan(a['centers'][1]).all() and a['inertia'][1] == 0.0
    outs = _frames_of(a)
    for f, velo in enumerate(frames):
        one = _batch([velo], 16, 3)
        assert outs[f].tobytes() == one['velo'].tobytes(), f
        for key in ('centers', 'inertia', 'group_sizes'):
            assert a[key][f].tobytes() == one[key][0].tobytes(), (f, key)


def test_short_frame_raises_and_next_call_succeeds():
    frames = [obd.velodyne_frame(21, 1000, full_360=False), obd.velodyne_frame(22, 1000, full_360=False)[:10]]
    with pytest.raises(ValueError, match='frame 1 has 10 points'):
        _batch(frames, 64)
    res = _batch(frames[:1], 64)
    assert res['velo'].shape[0] > 0
    with pytest.raises(ValueError):
        _batch(frames, 0)


def _training_tree(root, seeds, num_points):
    names = ok.write_synthetic_kitti(root, seeds, num_points=num_points, test_split=False)
    os.makedirs(os.path.join(root, '3DOP_splits'))
    with open(os.path.join(root, '3DOP_splits', 'val.txt'), 'w') as f:
        f.write(''.join(n + '\n' for n in names))
    return names


def test_cli_writes_batch_api_bytes_for_any_batch_size(tmp_path):
    from pointgnn_b200.scripts import point_cloud_downsample as pcd
    root = str(tmp_path / 'kitti')
    names = _training_tree(root, [31, 32, 33, 34, 35], 3000)
    trees = {}
    for bs in (1, 5):
        out = str(tmp_path / ('out%d' % bs))
        pcd.main(['--dataset_root_dir', root, '--output_dir', out, '--batch_size', str(bs)])
        trees[bs] = {n: open(os.path.join(out, n + '.bin'), 'rb').read() for n in names}
    assert trees[1] == trees[5]
    velo = [np.fromfile(os.path.join(root, 'velodyne/training/velodyne', n + '.bin'), np.float32).reshape(-1, 4)
            for n in names]
    for n, out in zip(names, _frames_of(_batch(velo, 64))):
        assert trees[1][n] == out.tobytes(), n
    pcd.main(['--dataset_root_dir', root, '--batch_size', '2'])        # the reference's default output directory
    default = os.path.join(root, 'velodyne/training_downsampled_2/velodyne')
    assert {n: open(os.path.join(default, n + '.bin'), 'rb').read() for n in names} == trees[1]


def test_run_on_downsampled_tree(tmp_path):
    from pointgnn_b200 import run
    from pointgnn_b200.scripts import point_cloud_downsample as pcd
    from test_run_batched_gpu import _checkpoint
    root = str(tmp_path / 'kitti')
    names = _training_tree(root, [36, 37, 38], 6000)
    pcd.main(['--dataset_root_dir', root])
    sparse = str(tmp_path / 'kitti_sparse')
    for d in ('image', 'calib', '3DOP_splits'):
        shutil.copytree(os.path.join(root, d), os.path.join(sparse, d))
    shutil.copytree(os.path.join(root, 'velodyne/training_downsampled_2/velodyne'),
                    os.path.join(sparse, 'velodyne/training/velodyne'))
    ckpt = str(tmp_path / 'ckpt')
    _checkpoint(ckpt, 'i')
    out = str(tmp_path / 'results')
    run.main([ckpt, '--dataset_root_dir', sparse, '--output_dir', out, '--batch_size', '2'])
    for n in names:
        assert os.path.isfile(os.path.join(out, 'data', n + '.txt')), n

"""Beam downsampling without a GPU: the NumPy restatement of scripts/point_cloud_downsample.py against the bytes the
reference's own script wrote, the exact 1-D k-means against scikit-learn's fits and brute force, the sm_90a build of
pg_beam.cu without register spills, and the CLI's argument checks."""
import itertools
import os

import numpy as np
import pytest

import cuda_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, 'tests', 'golden', 'beam_downsample.npz'))


def _frames():
    return range(len(GOLDEN['names']))


@pytest.mark.parametrize('i', _frames())
def test_restatement_reproduces_reference_bytes(i):
    from oracle import beam_downsample as obd
    out = obd.downsample(GOLDEN['velo_%d' % i], GOLDEN['sk_centers'][i], int(GOLDEN['downsample_rate']))
    assert out.dtype == np.float32
    assert out.tobytes() == GOLDEN['bin_%d' % i].tobytes()


def test_cosine_dtype_chain():
    """float32 norm ((x*x + y*y) + z*z), float64 z / norm; a zero-norm point gives NaN and is never kept."""
    from oracle import beam_downsample as obd
    rng = np.random.default_rng(3)
    xyz = rng.normal(0, 20, (5000, 3)).astype(np.float32)
    xyz[7] = 0.0
    cos = obd.cosines(xyz)
    sq = xyz * xyz
    norm = np.sqrt((sq[:, 0] + sq[:, 1]) + sq[:, 2])
    assert norm.dtype == np.float32
    with np.errstate(invalid='ignore'):
        want = xyz[:, 2].astype(np.float64) / norm.astype(np.float64)
    assert np.array_equal(cos, want, equal_nan=True) and np.isnan(cos[7])
    assert not obd.band_mask(cos, np.linspace(-0.9, 0.9, 64), 1)[7]


@pytest.mark.parametrize('i', _frames())
def test_exact_kmeans_not_above_sklearn(i):
    from oracle import beam_downsample as obd
    cos = obd.cosines(GOLDEN['velo_%d' % i][:, :3])
    res = obd.exact_kmeans_1d(cos, int(GOLDEN['num_clusters']))
    assert res['inertia'] <= GOLDEN['sk_inertia'][i] * (1 + 1e-12)
    x = np.sort(cos)
    c = res['centers']
    bounds = np.concatenate([[0], np.cumsum(res['sizes'])])
    assert bounds[-1] == len(x) and (res['sizes'] > 0).all() and np.all(np.diff(c) >= 0)
    label = np.repeat(np.arange(len(c)), res['sizes'])           # contiguous in sorted order
    own = np.abs(x - c[label])
    assert (own <= np.abs(x[:, None] - c[None, :]).min(axis=1)).all()


def test_exact_kmeans_matches_brute_force():
    from oracle import beam_downsample as obd
    rng = np.random.default_rng(11)
    for t in range(40):
        n = int(rng.integers(2, 10))
        k = int(rng.integers(1, n + 1))
        x = rng.normal(size=n) if t % 3 else np.round(rng.normal(size=n))   # every third with duplicates
        best = min(sum(((g - g.mean()) ** 2).sum() for g in np.split(np.sort(x), cuts))
                   for cuts in itertools.combinations(range(1, n), k - 1))
        got = obd.exact_kmeans_1d(x, k)['inertia']
        assert abs(got - best) <= 1e-12 * best + 1e-15, (x, k, got, best)


def test_exact_kmeans_degenerate_frames():
    from oracle import beam_downsample as obd
    res = obd.exact_kmeans_1d(np.array([0.1, 0.1, -0.2, 0.3, 0.3, 0.1, np.nan]), 5)   # 3 distinct values, k = 5
    assert res['inertia'] == 0.0 and list(res['sizes']) == [1, 1, 1, 1, 2]   # ties: smallest split
    assert list(res['centers']) == [-0.2, 0.1, 0.1, 0.1, 0.3]
    with pytest.raises(ValueError):
        obd.exact_kmeans_1d(np.array([0.1, 0.2, np.nan, np.nan]), 3)
    assert np.isnan(obd.exact_kmeans_1d(np.array([np.nan]), 4)['centers']).all()


def test_beam_kernel_builds_without_spills():
    kernels = cuda_build.kernels('pg_beam.cu')
    assert 'pg_beam.cu' in cuda_build.make_var('SRCS').split()
    rows = [k for k in kernels.values() if 'beam_' in k.mangled]
    assert len(rows) == 12, [k.mangled for k in kernels.values()]
    assert all(k.spill_stores == 0 and k.spill_loads == 0 for k in rows), [(k.name, k.spill_stores, k.spill_loads)
                                                                           for k in rows]


@pytest.mark.parametrize('flag,value', [('--downsample_rate', '0'), ('--downsample_rate', '-2'),
                                        ('--num_clusters', '0'), ('--batch_size', '0')])
def test_cli_rejects_bad_arguments(capsys, flag, value):
    from pointgnn_b200.scripts import point_cloud_downsample as pcd
    with pytest.raises(SystemExit):
        pcd.main(['--dataset_root_dir', '/nonexistent', flag, value])
    assert flag in capsys.readouterr().err


def test_cli_defaults_are_the_reference_paths():
    from pointgnn_b200.scripts import point_cloud_downsample as pcd
    a = pcd.parse_args(['--dataset_root_dir', 'D'])
    assert (a.downsample_rate, a.num_clusters) == (2, 64)
    assert os.path.normpath(a.dataset_split_file) == os.path.normpath('D/3DOP_splits/val.txt')
    assert os.path.normpath(a.output_dir) == os.path.normpath('D/velodyne/training_downsampled_2/velodyne')
    a = pcd.parse_args(['--dataset_root_dir', 'D', '--downsample_rate', '4'])
    assert os.path.normpath(a.output_dir) == os.path.normpath('D/velodyne/training_downsampled_4/velodyne')

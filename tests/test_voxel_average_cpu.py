"""`downsample_by_voxel_size` without a GPU: the oracle's restatement of downsample_by_average_voxel against the
reference's own output (tests/golden/kitti_voxel_avg.npz, made by tools/make_golden.py kitti_voxel_avg), the error
cases, and the way run.py hands the config key to the input stage."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import kitti as ok
from oracle import voxel_average as ova

IO = dict(np.load(os.path.join(GOLDEN, 'kitti_io.npz')))
VA = dict(np.load(os.path.join(GOLDEN, 'kitti_voxel_avg.npz')))
CALIB = ok.parse_calib(os.path.join(GOLDEN, 'kitti_calib.txt'))
TAGS = {0.1: '0p1', 0.4: '0p4'}


@pytest.mark.parametrize('voxel_size', sorted(TAGS))
def test_restatement_matches_reference_voxels_and_means(voxel_size):
    tag = TAGS[voxel_size]
    cam, refl = ova.velo_to_cam(IO['velo'], CALIB)
    xyz, attr, keys, counts = ova.downsample_by_average_voxel(cam, refl, voxel_size)
    assert xyz.dtype == np.float32 and attr.dtype == np.float32
    assert np.array_equal(keys, VA['keys_' + tag]) and np.array_equal(counts, VA['counts_' + tag])
    assert np.all(np.diff(keys) > 0) and counts.sum() == len(cam) and counts.max() > 1
    assert np.abs(xyz - VA['mean_xyz_' + tag]).max() < 1e-4
    assert np.abs(attr - VA['mean_attr_' + tag]).max() < 1e-4


@pytest.mark.parametrize('voxel_size', sorted(TAGS))
def test_restated_input_stage_matches_reference_crop(voxel_size):
    tag = TAGS[voxel_size]
    h, w = IO['image'].shape[:2]
    xyz, attr, kept = ova.cam_points_in_image(IO['velo'], CALIB, w, h, voxel_size, IO['image'])
    want = VA['crop_index_' + tag]
    crop_unsure, pixel_unsure = VA['crop_unsure_' + tag], VA['pixel_unsure_' + tag]
    # the float32 rounding of a mean may only change the verdict of a point the fixture recorded as near a boundary
    assert set(np.setxor1d(kept, want)) <= set(crop_unsure)
    assert len(crop_unsure) <= 0.01 * len(want) and len(pixel_unsure) <= 0.05 * len(want)
    both, ours, theirs = np.intersect1d(kept, want, return_indices=True)
    assert len(both) >= 0.99 * len(want)
    assert np.abs(xyz[ours] - VA['crop_xyz_' + tag][theirs]).max() < 1e-4
    assert np.abs(attr[ours, 0] - VA['crop_attr_' + tag][theirs, 0]).max() < 1e-4
    sure = ~np.isin(both, pixel_unsure)
    assert sure.sum() >= 0.95 * len(both)
    assert np.array_equal(attr[ours][sure, 1:], VA['crop_attr_' + tag][theirs][sure, 1:].astype(np.float32))


def test_means_are_sums_in_point_order():
    # 1e8 + 1 - 1e8 style cancellation: only the index-order fp64 sum gives these bits
    xyz = np.array([[0.0, 0.0, 0.0], [0.01, 0.02, 0.03], [0.02, 0.01, 0.0], [5.0, 5.0, 5.0]], np.float32)
    attr = np.array([[1e8], [1.0], [-1e8], [0.5]], np.float32)
    out_xyz, out_attr, keys, counts = ova.downsample_by_average_voxel(xyz, attr, 0.1)
    assert counts.tolist() == [3, 1]
    want = ((np.float64(np.float32(1e8)) + 1.0) + np.float64(np.float32(-1e8))) / 3.0
    assert out_attr[0, 0] == np.float32(want) and out_attr[1, 0] == np.float32(0.5)
    assert np.array_equal(out_xyz[1], xyz[3])


def test_attr_is_optional_and_empty_frame_is_empty():
    xyz = np.random.default_rng(0).uniform(0, 3, (50, 3)).astype(np.float32)
    a = ova.downsample_by_average_voxel(xyz, None, 0.5)
    b = ova.downsample_by_average_voxel(xyz, xyz[:, :2], 0.5)
    assert a[1] is None and np.array_equal(a[0], b[0]) and b[1].shape == (len(b[0]), 2)
    out_xyz, out_attr, keys, counts = ova.downsample_by_average_voxel(np.zeros((0, 3), np.float32),
                                                                      np.zeros((0, 1), np.float32), 0.1)
    assert out_xyz.shape == (0, 3) and out_attr.shape == (0, 1) and len(keys) == 0 and len(counts) == 0


@pytest.mark.parametrize('voxel_size', [0.0, -0.1, float('nan'), float('inf')])
def test_bad_voxel_size_is_a_value_error(voxel_size):
    from pointgnn_b200 import _lib
    xyz = np.zeros((4, 3), np.float32)
    with pytest.raises(ValueError):
        ova.downsample_by_average_voxel(xyz, None, voxel_size)
    # the binding refuses it before it looks at the tensors: no device is needed to get here
    with pytest.raises(ValueError):
        _lib.voxel_average(torch.zeros(4, 3), None, torch.tensor([0, 4], dtype=torch.int32), voxel_size)


def test_key_overflow_is_a_value_error_not_a_wrap():
    xyz = np.array([[0.0, 0.0, 0.0], [3.0, 3.0, 3.0]], np.float32)
    ova.downsample_by_average_voxel(xyz, None, 0.0025)          # 1201^3 < 2^31: fine
    with pytest.raises(ValueError, match='int32 voxel key'):
        ova.downsample_by_average_voxel(xyz, None, 0.002)       # 1501^3 > 2^31 - 1


@pytest.mark.parametrize('config_value,want', [(0.1, 0.1), (None, None), ('absent', None)])
def test_run_hands_the_config_key_to_the_input_stage(monkeypatch, config_value, want):
    from pointgnn_b200 import run
    seen = {}

    def fake(velo, calib, size, image, device=None, downsample_voxel_size='unset'):
        seen.update(voxel=downsample_voxel_size, device=device, args=(velo, calib, size, image))
        return torch.zeros(2, 3), torch.ones(2, 1), torch.tensor([0, 2], dtype=torch.int32)

    monkeypatch.setattr(run.kitti_dataset, 'cam_points_in_image_batch', fake)
    config = {'input_features': 'i000'}
    if config_value != 'absent':
        config['downsample_by_voxel_size'] = config_value
    xyz, attr, frame_ptr = run.input_stage(config, 'velo', 'calib', 'size', None, torch.device('cpu'))
    assert seen['voxel'] == want and seen['args'] == ('velo', 'calib', 'size', None)
    assert attr.shape == (2, 4) and attr[:, 1:].abs().sum() == 0 and frame_ptr.tolist() == [0, 2]


def test_dataset_method_takes_the_voxel_size(monkeypatch):
    import inspect
    from pointgnn_b200.dataset import kitti_dataset
    assert 'downsample_voxel_size' in inspect.signature(kitti_dataset.cam_points_in_image_batch).parameters
    assert list(inspect.signature(kitti_dataset.downsample_by_average_voxel).parameters) == ['points', 'voxel_size']
    src = inspect.getsource(kitti_dataset.KittiDataset.get_cam_points_in_image_with_rgb)
    assert 'downsample_voxel_size=downsample_voxel_size' in src

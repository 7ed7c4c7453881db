"""pg_voxel_average and the input stage with `downsample_by_voxel_size` on the GPU.

The kernel follows the oracle's restatement (oracle/voxel_average.py: fp64 sums in point order, one rounding to
float32), so from the same float32 cloud the two must agree bit for bit; the reference's own float64 means
(tests/golden/kitti_voxel_avg.npz) are within 1e-4.  The camera transform of the GPU stage differs from the BLAS
product of the reference in the last bit of some coordinates (see test_kitti_gpu.py), which can move a point across
a voxel face: the comparison of the whole stage with the reference's cropped cloud therefore allows a few voxels
without a partner, and the whole stage is also checked bit for bit from the GPU's own transform."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import graph as ograph
from oracle import kitti as ok
from oracle import synth
from oracle import voxel_average as ova

pytestmark = pytest.mark.gpu
IO = dict(np.load(os.path.join(GOLDEN, 'kitti_io.npz')))
VA = dict(np.load(os.path.join(GOLDEN, 'kitti_voxel_avg.npz')))
CALIB_FILE = os.path.join(GOLDEN, 'kitti_calib.txt')
TAGS = {0.1: '0p1', 0.4: '0p4'}
CFG = 'car_auto_T3_train'


def _dev(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def _average(clouds, attrs, voxel_size):
    """pg_voxel_average on a batch of NumPy clouds -> (xyz, attr, frame_ptr) as NumPy."""
    from pointgnn_b200 import _lib
    fp = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)
    xyz, attr, out_fp = _lib.voxel_average(_dev(np.vstack(clouds), np.float32), _dev(np.vstack(attrs), np.float32),
                                           _dev(fp), voxel_size)
    return xyz.cpu().numpy(), attr.cpu().numpy(), out_fp.cpu().numpy()


def _same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


@pytest.mark.parametrize('voxel_size', sorted(TAGS))
def test_kernel_on_the_reference_frame(voxel_size):
    tag = TAGS[voxel_size]
    cam, refl = ova.velo_to_cam(IO['velo'], ok.parse_calib(CALIB_FILE))
    xyz, attr, fp = _average([cam], [refl], voxel_size)
    want_xyz, want_attr, keys, counts = ova.downsample_by_average_voxel(cam, refl, voxel_size)
    assert fp.tolist() == [0, len(VA['keys_' + tag])]
    assert _same_bits(xyz, want_xyz) and _same_bits(attr, want_attr)
    assert np.abs(xyz - VA['mean_xyz_' + tag]).max() < 1e-4 and np.abs(attr - VA['mean_attr_' + tag]).max() < 1e-4


@pytest.mark.parametrize('num_points', [20000, 120000])
@pytest.mark.parametrize('voxel_size', [0.05, 0.1, 0.4])
def test_kernel_matches_restatement_on_seeded_clouds(num_points, voxel_size):
    xyz, intensity = synth.lidar_frame(900 + num_points // 1000, num_points, full_360=num_points > 25000)
    attr = np.hstack([intensity, xyz[:, :1] * 0.5, -xyz[:, 1:2]]).astype(np.float32)      # three channels
    got_xyz, got_attr, fp = _average([xyz], [attr], voxel_size)
    want_xyz, want_attr, keys, counts = ova.downsample_by_average_voxel(xyz, attr, voxel_size)
    assert fp.tolist() == [0, len(keys)] and len(keys) < num_points
    assert _same_bits(got_xyz, want_xyz) and _same_bits(got_attr, want_attr)


def test_batch_equals_single_frame_calls_with_degenerate_frames():
    rng = np.random.default_rng(3)
    clouds = [synth.lidar_frame(70 + i, 3000 + 500 * i)[0] for i in range(8)]
    clouds[2] = np.array([[1.5, -2.0, 7.25]], np.float32)                                   # one point
    clouds[4] = np.zeros((0, 3), np.float32)                                                # empty, inside the batch
    clouds[6] = (np.array([[3.0, 1.0, 9.0]]) + rng.uniform(0, 0.09, (40, 3))).astype(np.float32)   # one voxel
    clouds[7] = np.zeros((0, 3), np.float32)                                                # empty, last
    attrs = [rng.uniform(0, 1, (len(c), 1)).astype(np.float32) for c in clouds]
    xyz, attr, fp = _average(clouds, attrs, 0.1)
    assert fp[0] == 0 and fp[-1] == len(xyz)
    for f, (c, a) in enumerate(zip(clouds, attrs)):
        want_xyz, want_attr, _, _ = ova.downsample_by_average_voxel(c, a, 0.1)
        assert _same_bits(xyz[fp[f]:fp[f + 1]], want_xyz) and _same_bits(attr[fp[f]:fp[f + 1]], want_attr), f
        if len(c):
            one_xyz, one_attr, one_fp = _average([c], [a], 0.1)
            assert _same_bits(one_xyz, want_xyz) and _same_bits(one_attr, want_attr) and one_fp.tolist() == [0, len(want_xyz)]
    assert fp[3] - fp[2] == 1 and _same_bits(xyz[fp[2]:fp[3]], clouds[2])
    assert fp[5] == fp[4] and fp[7] - fp[6] == 1 and fp[8] == fp[7]


def test_numpy_entry_point_and_errors():
    from pointgnn_b200 import _lib
    from pointgnn_b200.dataset import kitti_dataset
    xyz, intensity = synth.lidar_frame(11, 5000)
    out = kitti_dataset.downsample_by_average_voxel(kitti_dataset.Points(xyz=xyz, attr=intensity), 0.2)
    want_xyz, want_attr, _, _ = ova.downsample_by_average_voxel(xyz, intensity, 0.2)
    assert _same_bits(out.xyz, want_xyz) and _same_bits(out.attr, want_attr)
    no_attr = kitti_dataset.downsample_by_average_voxel(kitti_dataset.Points(xyz=xyz, attr=None), 0.2)
    assert no_attr.attr is None and _same_bits(no_attr.xyz, want_xyz)
    empty = kitti_dataset.downsample_by_average_voxel(
        kitti_dataset.Points(xyz=np.zeros((0, 3), np.float32), attr=np.zeros((0, 1), np.float32)), 0.2)
    assert empty.xyz.shape == (0, 3) and empty.attr.shape == (0, 1)
    # second frame: 1501^3 voxels, where the reference's int32 key wraps
    far = np.array([[0.0, 0.0, 0.0], [3.0, 3.0, 3.0]], np.float32)
    fp = torch.tensor([0, 2, 4], dtype=torch.int32).cuda()
    with pytest.raises(ValueError, match='frame 1'):
        _lib.voxel_average(_dev(np.vstack([far * np.float32(0.1), far])), None, fp, 0.002)
    _lib.voxel_average(_dev(far), None, torch.tensor([0, 2], dtype=torch.int32).cuda(), 0.0025)      # 1201^3: fine
    with pytest.raises(ValueError):         # more than 65 536 voxels on one axis
        _lib.voxel_average(_dev(np.array([[0, 0, 0], [100.0, 0, 0]], np.float32)), None,
                           torch.tensor([0, 2], dtype=torch.int32).cuda(), 0.001)
    with pytest.raises(ValueError):
        _lib.voxel_average(_dev(xyz), None, torch.tensor([0, 5000], dtype=torch.int32).cuda(), float('nan'))


@pytest.mark.parametrize('voxel_size', sorted(TAGS))
def test_input_stage_with_downsampling(voxel_size):
    from scipy.spatial import cKDTree
    from pointgnn_b200 import _lib
    from pointgnn_b200.dataset import kitti_dataset
    tag = TAGS[voxel_size]
    calib = kitti_dataset.parse_calib(CALIB_FILE)
    h, w = IO['image'].shape[:2]
    frames = [IO['velo'], IO['velo'][::-1].copy()]
    xyz, attr, fp = kitti_dataset.cam_points_in_image_batch(frames, [calib] * 2, [(w, h)] * 2, [IO['image']] * 2,
                                                            downsample_voxel_size=voxel_size)
    xyz, attr, fp = xyz.cpu().numpy(), attr.cpu().numpy(), fp.cpu().numpy()
    # bit for bit from the GPU's own camera-frame points: the average, the crop and the colours
    cam, refl = _lib.velo_to_cam(_dev(np.vstack(frames)), torch.tensor([0, len(IO['velo']), 2 * len(IO['velo'])],
                                                                       dtype=torch.int32).cuda(),
                                 np.stack([calib['velo_to_cam'].astype(np.float32)] * 2))
    cam, refl = cam.cpu().numpy(), refl.cpu().numpy()
    for f in range(2):
        rows = slice(f * len(IO['velo']), (f + 1) * len(IO['velo']))
        a_xyz, a_refl, _, _ = ova.downsample_by_average_voxel(cam[rows], refl[rows], voxel_size)
        keep, img = ova.crop_mask(a_xyz, calib, w, h)
        u, v = img[keep, 0].astype(np.float32), img[keep, 1].astype(np.float32)
        rgb = IO['image'][np.int32(v), np.int32(u), ::-1].astype(np.float32) / 255
        assert _same_bits(xyz[fp[f]:fp[f + 1]], a_xyz[keep]), f
        assert _same_bits(attr[fp[f]:fp[f + 1]], np.hstack([a_refl[keep], rgb])), f
    # against the reference's cropped cloud: all but a few voxels have a partner within 1e-4, with its colours
    want_xyz, want_attr = VA['crop_xyz_' + tag], VA['crop_attr_' + tag]
    pixel_unsure = np.isin(VA['crop_index_' + tag], VA['pixel_unsure_' + tag])
    for f in range(2):
        got_xyz, got_attr = xyz[fp[f]:fp[f + 1]], attr[fp[f]:fp[f + 1]]
        assert abs(len(got_xyz) - len(want_xyz)) <= 0.005 * len(want_xyz)
        dist, nearest = cKDTree(got_xyz.astype(np.float64)).query(want_xyz)
        paired = dist < 1e-4
        assert paired.sum() >= 0.995 * len(want_xyz), (f, int(paired.sum()), len(want_xyz))
        assert np.abs(got_attr[nearest[paired], 0] - want_attr[paired, 0]).max() < 1e-4
        sure = paired & ~pixel_unsure
        assert np.array_equal(got_attr[nearest[sure], 1:], want_attr[sure, 1:].astype(np.float32))
    # reflectance only, through the dataset class of one frame
    single = kitti_dataset.cam_points_in_image_batch([IO['velo']], [calib], [(w, h)], downsample_voxel_size=voxel_size)
    assert _same_bits(single[0].cpu().numpy(), xyz[:fp[1]]) and _same_bits(single[1].cpu().numpy(), attr[:fp[1], :1])


def test_without_downsampling_the_fused_call_runs_unchanged():
    from pointgnn_b200 import _lib
    from pointgnn_b200.dataset import kitti_dataset
    calib = kitti_dataset.parse_calib(CALIB_FILE)
    h, w = IO['image'].shape[:2]
    frames = [IO['velo'], IO['velo'][::-1].copy()]
    for images in (None, [IO['image']] * 2):
        got = kitti_dataset.cam_points_in_image_batch(frames, [calib] * 2, [(w, h)] * 2, images, downsample_voxel_size=None)
        flat = offsets = None
        if images is not None:
            flat = _dev(np.concatenate([im.reshape(-1) for im in images]))
            offsets = np.array([0, IO['image'].size], np.int64)
        fp = torch.tensor([0, len(IO['velo']), 2 * len(IO['velo'])], dtype=torch.int32).cuda()
        want = _lib.cam_points_in_image(_dev(np.vstack(frames)), fp, np.stack([calib['velo_to_cam'].astype(np.float32)] * 2),
                                        np.stack([calib['cam_to_image']] * 2), np.array([(w, h)] * 2, np.int32), flat, offsets)
        for a, b in zip(got, want):
            assert _same_bits(a.cpu().numpy(), b.cpu().numpy())
        # and the two-call route without the averaging in between keeps and writes the same points
        cam, refl = _lib.velo_to_cam(_dev(np.vstack(frames)), fp, np.stack([calib['velo_to_cam'].astype(np.float32)] * 2))
        split = _lib.cam_points_crop(cam, refl, fp, np.stack([calib['cam_to_image']] * 2), np.array([(w, h)] * 2, np.int32),
                                     flat, offsets)
        for a, b in zip(split, want):
            assert _same_bits(a.cpu().numpy(), b.cpu().numpy())


def _checkpoint(path, voxel_size):
    os.makedirs(path)
    with open(os.path.join(GOLDEN, 'config_%s.json' % CFG)) as f:
        config = json.load(f)
    config['downsample_by_voxel_size'] = voxel_size
    with open(os.path.join(path, 'config'), 'w') as f:
        json.dump(config, f)
    w = dict(np.load(os.path.join(GOLDEN, 'weights_%s.npz' % CFG)))
    b = w['output/predictor/cls/fully_connected_1/biases'].copy()
    b[1:-1] += 7.0          # as tests/test_run_batched_gpu.py: the trained model does not fire on synthetic boxes
    w['output/predictor/cls/fully_connected_1/biases'] = b
    np.savez(os.path.join(path, 'weights.npz'), **w)
    return config


def _run(tmp_path, root, names, tag, voxel_size, batch_size):
    from pointgnn_b200 import run
    ckpt = str(tmp_path / ('ckpt_%s_%d' % (tag, batch_size)))
    _checkpoint(ckpt, voxel_size)
    out_dir = str(tmp_path / ('out_%s_%d' % (tag, batch_size)))
    run.main([ckpt, '--test', '--dataset_root_dir', root, '--output_dir', out_dir, '--batch_size', str(batch_size)])
    files = {}
    for name in names:
        with open(os.path.join(out_dir, 'data', name + '.txt'), 'rb') as f:
            files[name] = f.read()
    return files


def test_run_with_the_config_key_set(tmp_path):
    from pointgnn_b200.dataset import kitti_dataset
    from pointgnn_b200.models import graph_gen
    root = str(tmp_path / 'kitti')
    names = ok.write_synthetic_kitti(root, [41, 42, 43, 44, 45, 46, 47, 48, 49, 50], 6000)
    on1 = _run(tmp_path, root, names, 'on', 0.2, 1)
    on8 = _run(tmp_path, root, names, 'on', 0.2, 8)
    off = _run(tmp_path, root, names, 'off', None, 8)
    assert on1 == on8
    assert sum(text.count(b'\n') - 1 for text in on8.values()) > 0, 'no detection at all: the test would be vacuous'
    assert on8 != off, 'the key had no effect on the results'
    # the graph of the averaged cloud = the oracle's graph of the same float32 array
    config = _checkpoint(str(tmp_path / 'ckpt_graph'), 0.2)
    velo = np.fromfile(os.path.join(root, 'velodyne/testing/velodyne', names[0] + '.bin'), dtype=np.float32).reshape(-1, 4)
    calib = kitti_dataset.parse_calib(os.path.join(root, 'calib/testing/calib', names[0] + '.txt'))
    full = kitti_dataset.cam_points_in_image_batch([velo], [calib], [(1242, 375)])[0]
    xyz = kitti_dataset.cam_points_in_image_batch([velo], [calib], [(1242, 375)], downsample_voxel_size=0.2)[0].cpu().numpy()
    assert 0 < len(xyz) < 0.9 * len(full)
    kw = config['runtime_graph_gen_kwargs']
    graph = graph_gen.get_graph_generate_fn(config['graph_gen_method'])(xyz, **kw)
    _, _, edges = ograph.gen_multi_level_local_graph_v3(xyz, **kw)
    for got, want in zip(graph[2], edges):
        assert np.array_equal(got, want)

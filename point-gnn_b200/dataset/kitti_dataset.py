"""The part of the reference's ``dataset/kitti_dataset.py`` that inference touches (run.py:70-86, 210-215,
361-404), with the per-point work on the GPU.

* ``KittiDataset`` - same constructor and the methods run.py calls: ``num_files``, ``num_classes``,
  ``get_filename``, ``get_calib`` (kitti_dataset.py:483-522), ``get_image`` (:691-701), ``get_velo_points``
  (:587-609), ``get_cam_points_in_image_with_rgb`` (:666-689) -> GPU (``pg_cam_points_in_image``),
  ``cam_points_to_image`` (:1036-1052), ``box3d_to_normals`` (:923-946), ``sel_xyz_in_box3d`` (:969-988).
  The last three are the NumPy forms, as in the reference, that ``run.kitti_labels`` uses; ``run.py`` itself
  runs them for every detection of a batch on the GPU (``models.postprocess.kitti_rows``, ``pg_kitti_rows``).
  ``get_image_size`` reads an image's size from its PNG header, for input features without colour.
  Labels, augmentation, statistics and visualisation are training / tooling code: not built.
* ``Points`` - the reference's namedtuple (kitti_dataset.py:14).
* ``beam_downsample_batch`` - the beam downsampling of the reference's ``scripts/point_cloud_downsample.py`` on the GPU
  (``pg_beam_downsample``), with an exact 1-D k-means in place of its scikit-learn ``KMeans``.
* ``cam_points_in_image_batch`` - several frames in one GPU call, results staying on the device (what the
  batched ``run.py`` and the end-to-end bench use); with ``downsample_voxel_size`` the camera-frame cloud is averaged
  per voxel ahead of the crop, as ``get_cam_points`` does (kitti_dataset.py:624-626).
* ``downsample_by_average_voxel`` - kitti_dataset.py:16-48 on the GPU (``pg_voxel_average``) for one frame.
"""
import os
from collections import namedtuple
from os.path import isfile, join

import numpy as np
import torch

from .. import _lib

Points = namedtuple('Points', ['xyz', 'attr'])


def box3d_to_cam_points(label, expend_factor=(1.0, 1.0, 1.0)):
    """kitti_dataset.py:85-116."""
    yaw = label['yaw']
    r = np.array([[np.cos(yaw), 0, np.sin(yaw)], [0, 1, 0], [-np.sin(yaw), 0, np.cos(yaw)]])
    h = label['height']
    delta_h = h * (expend_factor[0] - 1)
    w = label['width'] * expend_factor[1]
    l = label['length'] * expend_factor[2]
    corners = np.array([[l / 2, delta_h / 2, w / 2], [l / 2, delta_h / 2, -w / 2], [-l / 2, delta_h / 2, -w / 2],
                        [-l / 2, delta_h / 2, w / 2], [l / 2, -h - delta_h / 2, w / 2], [l / 2, -h - delta_h / 2, -w / 2],
                        [-l / 2, -h - delta_h / 2, -w / 2], [-l / 2, -h - delta_h / 2, w / 2]])
    cam_points_xyz = corners.dot(np.transpose(r)) + np.array([label['x3d'], label['y3d'], label['z3d']])
    return Points(xyz=cam_points_xyz, attr=None)


def box3d_to_normals(label, expend_factor=(1.0, 1.0, 1.0)):
    """kitti_dataset.py:118-141 -> (normals [3,3], lower [3], upper [3])."""
    p = box3d_to_cam_points(label, expend_factor).xyz
    wx = p[[0], :] - p[[4], :]
    lx, ux = np.matmul(wx, p[4, :]), np.matmul(wx, p[0, :])
    wy = p[[0], :] - p[[1], :]
    ly, uy = np.matmul(wy, p[1, :]), np.matmul(wy, p[0, :])
    wz = p[[0], :] - p[[3], :]
    lz, uz = np.matmul(wz, p[3, :]), np.matmul(wz, p[0, :])
    return np.concatenate([wx, wy, wz], axis=0), np.concatenate([lx, ly, lz]), np.concatenate([ux, uy, uz])


def sel_xyz_in_box3d(label, xyz, expend_factor=(1.0, 1.0, 1.0)):
    """kitti_dataset.py:143-162."""
    normals, lower, upper = box3d_to_normals(label, expend_factor)
    projected = np.matmul(xyz, np.transpose(normals))
    inside = [np.logical_and(projected[:, i] > lower[i], projected[:, i] < upper[i]) for i in range(3)]
    return np.logical_and.reduce(inside)


def parse_calib(calib_file):
    """KittiDataset.get_calib (kitti_dataset.py:483-522) for one calibration file."""
    with open(calib_file, 'r') as f:
        calib = {}
        for line in f:
            fields = line.split(' ')
            matrix_name = fields[0].rstrip(':')
            if matrix_name.strip() == '':
                continue
            calib[matrix_name] = np.array(fields[1:], dtype=np.float32)
    calib['P2'] = calib['P2'].reshape(3, 4)
    calib['R0_rect'] = calib['R0_rect'].reshape(3, 3)
    calib['Tr_velo_to_cam'] = calib['Tr_velo_to_cam'].reshape(3, 4)
    r0_rect = np.eye(4)
    r0_rect[:3, :3] = calib['R0_rect']
    calib['velo_to_rect'] = np.vstack([calib['Tr_velo_to_cam'], [0, 0, 0, 1]])
    calib['cam_to_image'] = np.hstack([calib['P2'][:, 0:3], [[0], [0], [0]]])
    calib['rect_to_cam'] = np.hstack([calib['R0_rect'],
                                      np.matmul(np.linalg.inv(calib['P2'][:, 0:3]), calib['P2'][:, [3]])])
    calib['rect_to_cam'] = np.vstack([calib['rect_to_cam'], [0, 0, 0, 1]])
    calib['velo_to_cam'] = np.matmul(calib['rect_to_cam'], calib['velo_to_rect'])
    calib['cam_to_velo'] = np.linalg.inv(calib['velo_to_cam'])
    calib['velo_to_image'] = np.matmul(calib['cam_to_image'], calib['velo_to_cam'])
    assert np.isclose(calib['velo_to_image'],
                      np.matmul(np.matmul(calib['P2'], r0_rect), calib['velo_to_rect'])).all()
    return calib


def downsample_by_average_voxel(points, voxel_size):
    """kitti_dataset.py:16-48 on the GPU: one point per occupied voxel of ``points`` (one frame, NumPy ``Points``;
    ``attr`` may be None), in ascending voxel-key order, xyz and attr the voxel's means.  The means are float32 (fp64
    sums in point order, rounded once) where the reference returns float64 from float32 sums of unspecified order; they
    agree within 1e-4.  Raises ValueError for a voxel size that is not positive and finite, or so small that the
    reference's int32 voxel key would wrap."""
    device = torch.device('cuda', torch.cuda.current_device())
    xyz = torch.from_numpy(np.ascontiguousarray(points.xyz, dtype=np.float32).reshape(-1, 3)).to(device)
    attr = None
    if points.attr is not None:
        attr = torch.from_numpy(np.ascontiguousarray(points.attr, dtype=np.float32)).to(device)      # [M, C]
    fp = torch.tensor([0, xyz.shape[0]], dtype=torch.int32, device=device)
    out_xyz, out_attr, _ = _lib.voxel_average(xyz, attr, fp, voxel_size)
    return Points(xyz=out_xyz.cpu().numpy(), attr=None if out_attr is None else out_attr.cpu().numpy())


def cam_points_in_image_batch(velo_list, calib_list, image_size_list, image_list=None, device=None,
                              downsample_voxel_size=None):
    """Several frames in ONE GPU call.  velo_list: [Mi,4] float32 arrays (the .bin contents); calib_list: dicts of
    ``parse_calib``; image_size_list: (width, height); image_list: optional BGR uint8 images (for rgb attributes);
    downsample_voxel_size: None, or the voxel edge of ``downsample_by_average_voxel``, applied to every frame's
    camera-frame cloud before the crop (three calls then: transform, average, crop).
    -> (xyz [N,3] CUDA, attr [N,1|4] CUDA, frame_ptr [F+1] CUDA int32)."""
    device = device or torch.device('cuda', torch.cuda.current_device())
    sizes = [v.shape[0] for v in velo_list]
    fp = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    velo = torch.from_numpy(np.ascontiguousarray(np.vstack(velo_list), dtype=np.float32)).to(device)
    vtc = np.stack([c['velo_to_cam'].astype(np.float32) for c in calib_list])
    cti = np.stack([np.asarray(c['cam_to_image'], dtype=np.float64) for c in calib_list])
    images = offsets = None
    if image_list is not None:
        flat = [np.ascontiguousarray(im, dtype=np.uint8).reshape(-1) for im in image_list]
        offsets = np.concatenate([[0], np.cumsum([f.size for f in flat])[:-1]]).astype(np.int64)
        images = torch.from_numpy(np.concatenate(flat)).to(device)
    fp = torch.from_numpy(fp).to(device)
    wh = np.asarray(image_size_list, np.int32)
    if downsample_voxel_size is None:
        return _lib.cam_points_in_image(velo, fp, vtc, cti, wh, images, offsets)
    xyz, refl = _lib.velo_to_cam(velo, fp, vtc)
    xyz, refl, fp = _lib.voxel_average(xyz, refl, fp, downsample_voxel_size)
    return _lib.cam_points_crop(xyz, refl, fp, cti, wh, images, offsets)


def beam_downsample_batch(velo, frame_ptr=None, downsample_rate=2, num_clusters=64, centers=None):
    """The beam downsampling of scripts/point_cloud_downsample.py:19-53 on the GPU (``pg_beam_downsample``): keep every
    ``downsample_rate``-th of ``num_clusters`` beam bands of each frame, the bands cut between the cluster centres
    of the points' zenith cosines.  The centres come from the exact 1-D k-means of each frame (deterministic; its
    inertia is never above a KMeans fit's), or from ``centers``.  Points with a zero norm are never kept.

    * ``velo`` a CUDA float32 [M, 4] tensor (x, y, z, reflectance) with ``frame_ptr`` [F+1] CUDA int32, ``centers``
      None or [F, K] CUDA float64 -> the dict of ``_lib.beam_downsample``: device tensors ``velo`` [R, 4] (kept rows,
      original order), ``frame_ptr`` [F+1], ``centers`` [F, K], and without ``centers`` also ``inertia`` [F] and
      ``group_sizes`` [F, K].
    * ``velo`` one frame's NumPy [M, 4] float32 array (``frame_ptr`` None), ``centers`` None or [K] -> (kept rows
      [R, 4] float32 array, centres [K] float64 array, inertia float or None).
    Raises ValueError for a frame with at least one but fewer than ``num_clusters`` clusterable points."""
    if frame_ptr is not None:
        return _lib.beam_downsample(velo, frame_ptr, num_clusters, downsample_rate, centers_in=centers)
    device = torch.device('cuda', torch.cuda.current_device())
    arr = np.ascontiguousarray(velo, dtype=np.float32).reshape(-1, 4)
    fp = torch.tensor([0, arr.shape[0]], dtype=torch.int32, device=device)
    cin = None
    if centers is not None:
        cin = torch.from_numpy(np.asarray(centers, dtype=np.float64).reshape(1, -1)).to(device)
    res = _lib.beam_downsample(torch.from_numpy(arr).to(device), fp, num_clusters, downsample_rate, centers_in=cin)
    inertia = float(res['inertia'][0]) if 'inertia' in res else None
    return res['velo'].cpu().numpy(), res['centers'][0].cpu().numpy(), inertia


class KittiDataset(object):
    """kitti_dataset.py:184-216 (inference subset)."""

    def __init__(self, image_dir, point_dir, calib_dir, label_dir, index_filename=None, is_training=True,
                 is_raw=False, difficulty=-100, num_classes=8):
        self._image_dir = image_dir
        self._point_dir = point_dir
        self._calib_dir = calib_dir
        self._label_dir = label_dir
        self._index_filename = index_filename
        if index_filename:
            self._file_list = self._read_index_file(index_filename)
        else:
            self._file_list = self._get_file_list(self._image_dir)
        self._verify_file_list(image_dir, point_dir, label_dir, calib_dir, self._file_list, is_training, is_raw)
        self._is_training = is_training
        self._is_raw = is_raw
        self.num_classes = num_classes
        self.difficulty = difficulty

    @property
    def num_files(self):
        return len(self._file_list)

    @staticmethod
    def _read_index_file(index_filename):
        with open(index_filename, 'r') as f:
            return [line.rstrip('\n').split('.')[0] for line in f]

    @staticmethod
    def _get_file_list(image_dir):
        return sorted(f.split('.')[0] for f in os.listdir(image_dir) if isfile(join(image_dir, f)))

    @staticmethod
    def _verify_file_list(image_dir, point_dir, label_dir, calib_dir, file_list, is_training, is_raw):
        for f in file_list:
            assert isfile(join(image_dir, f) + '.png'), 'Image %s does not exist' % (join(image_dir, f) + '.png')
            assert isfile(join(point_dir, f) + '.bin'), 'Point %s does not exist' % (join(point_dir, f) + '.bin')
            if not is_raw:
                assert isfile(join(calib_dir, f) + '.txt'), 'Calib %s does not exist' % (join(calib_dir, f) + '.txt')
            if is_training:
                assert isfile(join(label_dir, f) + '.txt'), 'Label %s does not exist' % (join(label_dir, f) + '.txt')

    def get_filename(self, frame_idx):
        return self._file_list[frame_idx]

    def get_calib(self, frame_idx):
        return parse_calib(join(self._calib_dir, self._file_list[frame_idx]) + '.txt')

    def get_image(self, frame_idx):
        import cv2
        return cv2.imread(join(self._image_dir, self._file_list[frame_idx]) + '.png')

    def get_image_size(self, frame_idx):
        """(height, width) of the frame's PNG, as ``get_image(frame_idx).shape[:2]``, read from the IHDR chunk that
        opens every PNG file instead of decoding the image."""
        path = join(self._image_dir, self._file_list[frame_idx]) + '.png'
        with open(path, 'rb') as f:
            head = f.read(24)
        # 8-byte signature, then the IHDR chunk: length (4), type (4), width (4), height (4), big-endian
        if len(head) < 24 or head[:8] != b'\x89PNG\r\n\x1a\n' or head[12:16] != b'IHDR':
            raise ValueError('%s is not a PNG file' % path)
        return int.from_bytes(head[20:24], 'big'), int.from_bytes(head[16:20], 'big')

    def get_velo_data(self, frame_idx):
        """The raw [M, 4] float32 content of the frame's .bin file (x, y, z, reflectance)."""
        return np.fromfile(join(self._point_dir, self._file_list[frame_idx]) + '.bin', dtype=np.float32).reshape(-1, 4)

    def get_velo_points(self, frame_idx, xyz_range=None):
        """kitti_dataset.py:587-609."""
        velo_data = self.get_velo_data(frame_idx)
        velo_points, reflections = velo_data[:, :3], velo_data[:, [3]]
        if xyz_range is not None:
            x_range, y_range, z_range = xyz_range
            mask = (velo_points[:, 0] > x_range[0]) * (velo_points[:, 0] < x_range[1])
            mask *= (velo_points[:, 1] > y_range[0]) * (velo_points[:, 1] < y_range[1])
            mask *= (velo_points[:, 2] > z_range[0]) * (velo_points[:, 2] < z_range[1])
            return Points(xyz=velo_points[mask], attr=reflections[mask])
        return Points(xyz=velo_points, attr=reflections)

    def get_cam_points_in_image_with_rgb(self, frame_idx, downsample_voxel_size=None, calib=None, xyz_range=None):
        """kitti_dataset.py:666-689 on the GPU -> Points(xyz [N,3], attr [N,4] = reflectance, r, g, b) as NumPy."""
        if xyz_range is not None:
            raise NotImplementedError('xyz_range is not used by run.py')
        if calib is None:
            calib = self.get_calib(frame_idx)
        image = self.get_image(frame_idx)
        xyz, attr, _ = cam_points_in_image_batch([self.get_velo_data(frame_idx)], [calib],
                                                 [(image.shape[1], image.shape[0])], [image],
                                                 downsample_voxel_size=downsample_voxel_size)
        return Points(xyz=xyz.cpu().numpy(), attr=attr.cpu().numpy())

    def cam_points_to_image(self, points, calib):
        """kitti_dataset.py:1036-1052."""
        cam_points_xyz1 = np.hstack([points.xyz, np.ones([points.xyz.shape[0], 1])])
        img_points_xyz = np.matmul(cam_points_xyz1, np.transpose(calib['cam_to_image']))
        return Points(img_points_xyz / img_points_xyz[:, [2]], points.attr)

    def box3d_to_normals(self, label, expend_factor=(1.0, 1.0, 1.0)):
        return box3d_to_normals(label, expend_factor)

    def sel_xyz_in_box3d(self, label, xyz, expend_factor=(1.0, 1.0, 1.0)):
        return sel_xyz_in_box3d(label, xyz, expend_factor)

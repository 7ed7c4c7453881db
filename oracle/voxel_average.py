"""CPU oracle for the `downsample_by_voxel_size` input path: the reference's ``downsample_by_average_voxel``
(dataset/kitti_dataset.py:16-48) as ``get_cam_points`` applies it (:611-627), ahead of the image crop (:666-689).

TEST INFRASTRUCTURE (see oracle/__init__.py).

The restatement keeps what the reference's code fixes - which points share a voxel (NumPy float32 ``//`` from the
frame minimum), the number of voxels, their ascending-key order - and replaces what it leaves open:

* the reference adds float32 values with ``np.add.reduceat`` in ``np.argsort(keys)`` order.  That sort is not stable,
  so the order of addition inside a voxel is unspecified.  Here: float64 sums in ascending point index.
* ``float32 / int64`` makes the reference's means float64 and everything after them runs on float64.  Here the float64
  mean is rounded once to float32, and the crop, the colour lookup and the graph see that float32 array.

The means of the two agree within 1e-4 (tests/golden/kitti_voxel_avg.npz holds the reference's).  The CUDA path
(pg_voxel_average) follows the same two rules, so it is compared with this file bit for bit.

The reference's int32 key wraps when dim_x * dim_y * dim_z exceeds 2^31 - 1; that is a ValueError here, as is a voxel
size that is not positive and finite.
"""
import math

import numpy as np

INT32_MAX = 2 ** 31 - 1


def voxel_keys(xyz, voxel_size):
    """kitti_dataset.py:23-30 -> (keys [M] int64, dims [3]) of a float32 cloud with at least one point."""
    offset = np.amin(xyz, axis=0, keepdims=True)
    idx = ((xyz - offset) // np.float32(voxel_size)).astype(np.int32).astype(np.int64)
    dims = np.amax(idx, axis=0) + 1
    if int(dims[0]) * int(dims[1]) * int(dims[2]) > INT32_MAX:
        raise ValueError('%d x %d x %d voxels of size %g: more than the 2^31 - 1 an int32 voxel key can number'
                         % (dims[0], dims[1], dims[2], voxel_size))
    return idx[:, 0] + idx[:, 1] * dims[0] + idx[:, 2] * dims[1] * dims[0], dims


def downsample_by_average_voxel(xyz, attr, voxel_size):
    """One frame.  xyz [M,3] float32, attr [M,C] float32 or None -> (xyz [V,3] float32, attr [V,C] float32 or None,
    keys [V] int64 ascending, counts [V] int64)."""
    voxel_size = float(voxel_size)
    if not (voxel_size > 0.0 and math.isfinite(voxel_size)):
        raise ValueError('voxel_size must be positive and finite, got %r' % voxel_size)
    xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    if xyz.shape[0] == 0:
        empty = None if attr is None else np.zeros((0,) + np.shape(attr)[1:], np.float32)
        return np.zeros((0, 3), np.float32), empty, np.zeros(0, np.int64), np.zeros(0, np.int64)
    keys, _ = voxel_keys(xyz, voxel_size)
    order = np.argsort(keys, kind='stable')           # inside a voxel: ascending point index
    unique_keys, start, counts = np.unique(keys[order], return_index=True, return_counts=True)
    values = xyz if attr is None else np.hstack([xyz, np.asarray(attr, dtype=np.float32).reshape(len(xyz), -1)])
    values = values[order].astype(np.float64)
    sums = np.zeros((len(unique_keys), values.shape[1]), np.float64)
    for k in range(int(counts.max())):                # the k-th point of every voxel that has one: sequential sums
        has = counts > k
        sums[has] += values[start[has] + k]
    means = (sums / counts[:, None].astype(np.float64)).astype(np.float32)
    return means[:, :3], (None if attr is None else means[:, 3:]), unique_keys.astype(np.int64), counts.astype(np.int64)


def velo_to_cam(velo_data, calib):
    """velo_points_to_cam (kitti_dataset.py:998-1006) on the raw [M,4] array -> (xyz [M,3] float32, attr [M,1])."""
    cam = np.matmul(velo_data[:, :3], np.transpose(calib['velo_to_cam'])[:3, :3].astype(np.float32))
    cam += np.transpose(calib['velo_to_cam'])[[3], :3].astype(np.float32)
    return cam, velo_data[:, [3]]


def crop_mask(cam, calib, width, height):
    """kitti_dataset.py:674-686 -> (keep [N] bool, projections [N,3] float64) of camera-frame points."""
    cam = np.asarray(cam, dtype=np.float64)      # the front test too is a float64 comparison on the means
    img = np.matmul(np.hstack([cam, np.ones([cam.shape[0], 1])]), np.transpose(calib['cam_to_image']))
    with np.errstate(divide='ignore', invalid='ignore'):
        img = img / img[:, [2]]
    keep = np.logical_and.reduce([cam[:, 2] > 0.1, img[:, 0] > 0, img[:, 0] < width, img[:, 1] > 0, img[:, 1] < height])
    return keep, img


def cam_points_in_image(velo_data, calib, width, height, voxel_size, image=None):
    """get_cam_points_in_image_with_rgb(frame, voxel_size) under the two rules above, from the raw [M,4] velodyne array
    -> (xyz [N,3] float32, attr [N,1] or [N,4] float32, kept [N] = ranks of the surviving voxels)."""
    cam, refl = velo_to_cam(velo_data, calib)
    cam, refl, _, _ = downsample_by_average_voxel(cam, refl, voxel_size)
    keep, img = crop_mask(cam, calib, width, height)
    cam, attr, img = cam[keep], refl[keep], img[keep]
    if image is not None:
        # the colour lookup truncates the float32 projection, as the GPU stage stores it
        u, v = img[:, 0].astype(np.float32), img[:, 1].astype(np.float32)
        rgb = image[np.int32(v), np.int32(u), ::-1].astype(np.float32) / 255
        attr = np.hstack([attr, rgb])
    return cam, attr, np.flatnonzero(keep)


def decision_margin(cam64, calib, width, height, radius=1e-4):
    """Which points' crop verdict / colour pixel could change when their coordinates move by up to ``radius``: evaluated
    at the eight corners of the cube of that half-edge around each float64 point.
    -> (crop_unsure [N] bool, pixel_unsure [N] bool)."""
    keep0, img0 = crop_mask(cam64, calib, width, height)
    with np.errstate(invalid='ignore'):
        pix0 = np.floor(img0[:, :2])
    crop_unsure = np.zeros(len(cam64), bool)
    pixel_unsure = np.zeros(len(cam64), bool)
    for dx in (-radius, radius):
        for dy in (-radius, radius):
            for dz in (-radius, radius):
                keep, img = crop_mask(cam64 + np.array([dx, dy, dz]), calib, width, height)
                crop_unsure |= keep != keep0
                with np.errstate(invalid='ignore'):
                    pixel_unsure |= np.any(np.floor(img[:, :2]) != pix0, axis=1)
    return crop_unsure, pixel_unsure & keep0

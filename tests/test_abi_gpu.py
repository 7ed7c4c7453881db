"""GPU tests of the drop-in boundary: every pointer argument is checked against the type the header declares for it."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_pointer_arguments_follow_the_declared_type():
    """A device pointer given a tensor of the wrong dtype, a NumPy array or a strided view, and a host pointer given an
    array of the wrong dtype, raise an error that names the parameter before the library runs."""
    from pointgnn_b200 import _lib
    params = torch.zeros((4, 3), dtype=torch.float32, device='cuda')
    indices = torch.zeros(2, dtype=torch.int32, device='cuda')
    with pytest.raises(TypeError, match='indices'):
        _lib.gather_rows(params, indices.long())
    with pytest.raises(TypeError, match='params'):
        _lib.gather_rows(params.double(), indices)
    with pytest.raises(ValueError, match='params'):
        _lib.gather_rows(params.t(), indices)
    out = torch.empty((2, 3), dtype=torch.float32, device='cuda')
    with pytest.raises(TypeError, match='params'):
        _lib._call('pg_gather_rows', params=params.cpu().numpy(), num_rows=4, num_channels=3, indices=indices,
                   num_indices=2, out=out)
    k = ctypes.c_int64(0)
    fp = torch.tensor([0, 4], dtype=torch.int32, device='cuda')
    keypoints = dict(xyz=params, frame_ptr=fp, num_frames=1, num_points=4, out_keypoint_idx=indices, capacity=2,
                     out_kp_frame_ptr=fp, out_num_keypoints_host=ctypes.byref(k))
    with pytest.raises(TypeError, match='voxel_size_host'):
        _lib._call('pg_voxel_keypoints', voxel_size_host=np.ones(3, np.float32), **keypoints)
    with pytest.raises(TypeError, match='out_num_keypoints_host'):
        _lib._call('pg_voxel_keypoints', voxel_size_host=np.ones(3), **dict(keypoints, out_num_keypoints_host=k))
    assert _lib.gather_rows(params, indices).shape == (2, 3)

"""Host side of the batched run.py (no GPU needed): image sizes from the PNG header, the --batch_size check, and
the Makefile build of pg_kitti.cu without register spills."""
import numpy as np
import pytest

import cuda_build


@pytest.mark.parametrize('width,height', [(1242, 375), (1224, 370), (1238, 374), (1241, 376)])
def test_image_size_from_png_header(tmp_path, width, height):
    import cv2
    from pointgnn_b200.dataset.kitti_dataset import KittiDataset
    for d in ('image', 'velodyne'):
        (tmp_path / d).mkdir()
    img = np.random.default_rng(width).integers(0, 255, (height, width, 3), dtype=np.uint8)
    cv2.imwrite(str(tmp_path / 'image' / '000007.png'), img)
    (tmp_path / 'velodyne' / '000007.bin').write_bytes(b'')
    ds = KittiDataset(str(tmp_path / 'image'), str(tmp_path / 'velodyne'), '', '', is_training=False, is_raw=True)
    assert ds.get_image_size(0) == cv2.imread(str(tmp_path / 'image' / '000007.png')).shape[:2] == (height, width)
    (tmp_path / 'image' / '000007.png').write_bytes(b'GIF89a' + bytes(40))
    with pytest.raises(ValueError):
        ds.get_image_size(0)


def test_batch_size_must_be_positive(capsys):
    from pointgnn_b200 import run
    with pytest.raises(SystemExit):
        run.main(['/nonexistent', '--batch_size', '0'])
    assert '--batch_size' in capsys.readouterr().err


def test_kitti_rows_kernel_builds_without_spills():
    kernels = cuda_build.kernels('pg_kitti.cu')
    assert 'pg_kitti.cu' in cuda_build.make_var('SRCS').split()
    rows = [k for k in kernels.values() if 'kitti_rows' in k.mangled]
    assert len(rows) == 2, [k.mangled for k in kernels.values()]
    assert all(k.spill_stores == 0 and k.spill_loads == 0 for k in rows), [(k.name, k.spill_stores, k.spill_loads)
                                                                           for k in rows]

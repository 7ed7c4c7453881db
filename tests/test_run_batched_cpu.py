"""Host side of the batched run.py (no GPU needed): image sizes from the PNG header, the --batch_size check, and
the Makefile build of pg_kitti.cu without register spills."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from test_kernel_build_cpu import CSRC, _make_var


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


def test_kitti_rows_kernel_builds_without_spills(tmp_path):
    if shutil.which('make') is None:
        pytest.skip('make not found')
    nvcc = _make_var('NVCC')
    if not (os.path.isfile(nvcc) or shutil.which(nvcc)):
        pytest.skip('nvcc not found')
    assert 'pg_kitti.cu' in _make_var('SRCS').split()
    flags = _make_var('NVCCFLAGS').split()
    res = subprocess.run([nvcc] + flags + ['-c', 'pg_kitti.cu', '-o', str(tmp_path / 'pg_kitti.o')], cwd=CSRC,
                         capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log[-4000:]
    props = re.findall(r'Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                       r'(\d+) bytes spill loads', log)
    rows = [p for p in props if 'kitti_rows' in p[0]]
    assert len(rows) == 2, [p[0] for p in props]
    assert all(p[2] == '0' and p[3] == '0' for p in rows), rows

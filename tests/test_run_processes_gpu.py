"""run.py --processes N on the synthetic KITTI-format tree of tests/test_run_batched_gpu.py: the same result files and
timer names as one process, and a failing rank that stops the job.

Five frames.  Every run's ranks share device 0 when the machine has one GPU (rank r runs on r % device count), so
these tests need no second device."""
import multiprocessing
import os

import numpy as np
import pytest

from test_run_batched_gpu import TIMERS, _checkpoint, _tree

pytestmark = pytest.mark.gpu


def _main(run, root, ckpt, out_dir, processes, batch_size):
    return run.main([ckpt, '--test', '--dataset_root_dir', root, '--output_dir', out_dir,
                     '--batch_size', str(batch_size), '--processes', str(processes)])


def _files(out_dir):
    data = os.path.join(out_dir, 'data')
    out = {}
    for name in sorted(os.listdir(data)):
        with open(os.path.join(data, name), 'rb') as f:
            out[name] = f.read()
    return out


def test_processes_write_the_files_of_one_process(tmp_path):
    from pointgnn_b200 import run
    root = str(tmp_path / 'kitti')
    names = _tree(root)
    ckpt = str(tmp_path / 'ckpt')
    _checkpoint(ckpt, 'i')
    files = {}
    # (processes, batch_size); the last run has more processes than frames, so ranks 5 and 6 have none
    for processes, batch_size in [(1, 1), (1, 3), (2, 1), (2, 3), (len(names) + 2, 3)]:
        out_dir = str(tmp_path / ('out_p%d_b%d' % (processes, batch_size)))
        times = _main(run, root, ckpt, out_dir, processes, batch_size)
        assert set(times) == TIMERS, (processes, batch_size, sorted(times))
        assert all(seconds >= 0 for seconds in times.values()) and times['total'] > 0, times
        files[processes, batch_size] = _files(out_dir)
        assert multiprocessing.active_children() == []
    want = files[1, 1]
    assert sorted(want) == [name + '.txt' for name in names]
    assert sum(text.count(b'\n') - 1 for text in want.values()) > 0, 'no detection at all: the test would be vacuous'
    for key, got in files.items():
        assert sorted(got) == sorted(want), key
        for name in want:
            assert got[name] == want[name], (key, name)


def test_failing_rank_stops_the_job(tmp_path):
    """A velodyne file of 5 float32 values makes its rank's reader raise ValueError (reshape(-1, 4)); main raises
    naming that rank, and no worker process outlives it."""
    from pointgnn_b200 import run
    root = str(tmp_path / 'kitti')
    names = _tree(root)
    ckpt = str(tmp_path / 'ckpt')
    _checkpoint(ckpt, 'i')
    bad = 3                                       # position 3 of the split: rank 1 of 2
    np.arange(5, dtype=np.float32).tofile(os.path.join(root, 'velodyne/testing/velodyne', names[bad] + '.bin'))
    with pytest.raises(RuntimeError, match='rank 1 of 2') as failure:
        _main(run, root, ckpt, str(tmp_path / 'out'), 2, 1)
    assert 'ValueError' in str(failure.value) and 'reshape' in str(failure.value), str(failure.value)
    assert multiprocessing.active_children() == []

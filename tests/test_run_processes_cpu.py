"""Host side of run.py --processes (no GPU needed): how the ranks split the frames into batches, how their timers
merge, and the checks the parent makes before it spawns a rank."""
import json
import multiprocessing

import pytest


def _batching_today(num_frames, batch_size):
    """run.py's batches before --processes: consecutive frames, the last batch possibly shorter."""
    return [list(range(first, min(first + batch_size, num_frames))) for first in range(0, num_frames, batch_size)]


@pytest.mark.parametrize('num_frames,batch_size,world', [(7, 3, 1), (7, 3, 2), (7, 3, 3), (7, 3, 4), (5, 3, 8),
                                                         (5, 1, 8), (0, 2, 3)])
def test_rank_batches_cover_every_frame_once(num_frames, batch_size, world):
    from pointgnn_b200.run import rank_batches
    from pointgnn_b200.utils.sharding import frames_for_rank
    seen = []
    for rank in range(world):
        batches = rank_batches(num_frames, batch_size, rank, world)
        assert all(1 <= len(b) <= batch_size for b in batches), batches
        assert all(len(b) == batch_size for b in batches[:-1]), batches
        assert sum(batches, []) == frames_for_rank(num_frames, rank, world)
        seen += sum(batches, [])
    assert sorted(seen) == list(range(num_frames))


@pytest.mark.parametrize('num_frames', [0, 1, 5, 7, 16, 3769])
@pytest.mark.parametrize('batch_size', [1, 3, 8])
def test_rank_batches_of_one_rank_are_todays_batches(num_frames, batch_size):
    from pointgnn_b200.run import rank_batches
    assert rank_batches(num_frames, batch_size, 0, 1) == _batching_today(num_frames, batch_size)


def test_rank_times_merge_stages_by_sum_and_total_by_max():
    from pointgnn_b200.run import merge_rank_times
    ranks = [{'fetch input': 1.0, 'gnn inference': 2.0, 'total': 5.0},
             {},                                   # a rank without frames
             {'fetch input': 0.5, 'gnn inference': 4.0, 'total': 7.0}]
    merged = merge_rank_times(ranks)
    assert list(merged) == ['fetch input', 'gnn inference', 'total']
    assert merged == {'fetch input': 1.5, 'gnn inference': 6.0, 'total': 7.0}


@pytest.mark.parametrize('processes', ['0', '-2'])
def test_processes_must_be_positive(capsys, processes):
    from pointgnn_b200 import run
    with pytest.raises(SystemExit):
        run.main(['/nonexistent', '--processes', processes])
    assert '--processes' in capsys.readouterr().err


def _no_spawn(args):
    raise AssertionError('a rank was spawned before the command line and the config were checked')


def test_parent_checks_before_spawning(tmp_path, monkeypatch, capsys):
    """The config assert, the codec check, -l and --batch_size fail in the parent, as with one process."""
    from pointgnn_b200 import run
    monkeypatch.setattr(run, 'run_ranks', _no_spawn)
    with pytest.raises(AssertionError, match='No config file'):
        run.main([str(tmp_path), '--processes', '2'])
    with pytest.raises(NotImplementedError):
        run.main([str(tmp_path), '--processes', '2', '-l', '1'])
    with pytest.raises(SystemExit):
        run.main([str(tmp_path), '--processes', '2', '--batch_size', '0'])
    assert '--batch_size' in capsys.readouterr().err
    with open(tmp_path / 'config', 'w') as f:
        json.dump({'box_encoding_method': 'direct_encoding'}, f)
    with pytest.raises(ValueError):
        run.main([str(tmp_path), '--processes', '2'])
    assert multiprocessing.active_children() == []

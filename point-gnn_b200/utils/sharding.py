"""Frame sharding across ranks (one process per GPU) and the counter exchange.

Frames are the independent units of the hot path (reference run.py:203: the loop body only
touches per-frame data; weights are read-only), so the multi-GPU plan is a pure partition:
frame ``i`` of the job goes to rank ``i % world`` (``frames_for_rank``), every rank runs the
same single-GPU path on its own frames, and the ONLY collective is an all-gather of a few
per-rank counters at the end (``gather_counters``): frames, device milliseconds, edges,
keypoints.  No feature / gradient / graph data ever crosses NVLink.

Backend-agnostic on purpose: ``nccl`` on the GPU machines, ``gloo`` in the CPU tests
(tests/test_sharding_cpu.py runs it with world_size 2).
"""
import torch
import torch.distributed as dist

COUNTER_NAMES = ('frames', 'device_ms', 'e2e_ms', 'edges0', 'edges1', 'keypoints')


def frames_for_rank(num_frames, rank, world):
    """Global frame ids owned by ``rank``: round-robin, so any prefix of the job is balanced."""
    if world < 1 or not 0 <= rank < world:
        raise ValueError('bad rank %r / world %r' % (rank, world))
    return list(range(rank, int(num_frames), world))


def frame_seed(step, slot, rank, frames_per_step):
    """Synthetic-frame seed of slot ``slot`` of step ``step`` on ``rank`` (rank-disjoint)."""
    return rank * 10000 + (step * frames_per_step + slot) % 10000


def gather_counters(counters, device=None):
    """All-gather ``counters`` (dict over COUNTER_NAMES) -> (per_rank [world, n] float64 CPU tensor,
    summary dict).  Times are reduced with MAX (the job ends when the slowest rank ends), counts
    with SUM.  Works without an initialised process group (world = 1)."""
    row = torch.tensor([float(counters.get(k, 0.0)) for k in COUNTER_NAMES], dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        rows = [torch.zeros_like(row) for _ in range(dist.get_world_size())]
        dist.all_gather(rows, row)
        per_rank = torch.stack(rows).cpu()
    else:
        per_rank = row[None, :].cpu()
    summary = {}
    for j, name in enumerate(COUNTER_NAMES):
        col = per_rank[:, j]
        summary[name] = float(col.max()) if name.endswith('_ms') else float(col.sum())
    return per_rank, summary


def throughput(summary, key='device_ms'):
    """Whole-job frames/s = frames of all ranks / time of the slowest rank."""
    ms = summary[key]
    return summary['frames'] / (ms * 1e-3) if ms > 0 else 0.0

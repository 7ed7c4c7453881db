"""The atomic-count model of tools/prof_segmax_carry.py on destination patterns that can be counted by hand: the
segment-max epilogue as it is (B = 1) and with a destination carry over blocks of B tiles."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import prof_segmax_carry as model  # noqa: E402

SLOTS = 66   # the car layer's CTA slots on 132 SMs (152 x 2)


def _flushes(dst, b, nd=None, slots=SLOTS):
    nd = int(np.max(dst)) + 1 if nd is None else nd
    return model.flushes(np.asarray(dst), nd, b, carry=True, slots=slots)


@pytest.mark.parametrize('b', [1, 2, 4, 8, 16])
def test_one_destination(b):
    # E = 64 x 4B rows (four blocks): each warp carries the one destination through its run of B sub-tiles and flushes
    # once per block, 4 warps x 4 blocks.  Without blocks: one flush per 16-row unit
    e = 64 * b * 4
    assert _flushes(np.zeros(e, int), b) == 16
    assert model.flushes(np.zeros(e, int), 1) == e // 16


def test_one_destination_consecutive_blocks_of_one_warpgroup():
    # one CTA slot: a warpgroup's next block is 3 on, so warp w of block 0 meets warp w of block 3: one destination
    # over 4 blocks of B = 2 flushes 4 warps x 3 warpgroups (the carry runs on from block 0 into block 3)
    assert _flushes(np.zeros(64 * 2 * 4, int), 2, slots=1) == 12


def test_degree_one():
    # no uniform unit: two halves of 8 runs each per 16 rows, whatever B
    for b in (1, 4, 16):
        assert _flushes(np.arange(160), b) == 160


def test_runs_ending_on_sub_tiles_and_blocks():
    # B = 2: warp w of block k owns the units 8k + 2w, 8k + 2w + 1.  Runs of 32 rows aligned to those pairs: one
    # flush each.  Shift by 16 rows: every run now spans two warps' units, two flushes each (no carry between warps)
    aligned = np.repeat(np.arange(8), 32)
    assert _flushes(aligned, 2) == 8
    shifted = np.concatenate([np.zeros(16, int), np.repeat(np.arange(1, 8), 32), np.full(16, 8)])
    assert _flushes(shifted, 2) == 1 + 7 * 2 + 1
    # B = 1: every 16-row unit flushes
    assert _flushes(aligned, 1) == 16


def test_mixed_unit_breaks_the_carry():
    # 40 rows of 0, 24 of 1: units 0, 1 uniform (0), unit 2 mixed (8 rows of 0, 8 of 1: two runs), unit 3 uniform (1)
    dst = np.concatenate([np.zeros(40, int), np.ones(24, int)])
    assert _flushes(dst, 4) == 1 + 2 + 1
    assert model.flushes(dst, 2) == 1 + 1 + 2 + 1


def test_tail_and_out_of_range_rows():
    # 20 rows: a uniform unit, then a tail unit of 4 valid rows (one run); an out-of-range destination is no flush
    assert _flushes(np.zeros(20, int), 4) == 1 + 1
    dst = np.zeros(32, int)
    dst[20] = 5
    # unit 1, first half: rows 16..19 and 21..23 are two runs around the out-of-range row 20; second half: one run
    assert model.flushes(dst, 1) == 1 + 3
    assert _flushes(dst, 4, nd=1) == 1 + 3


def test_b1_is_the_mapping_without_carry():
    rng = np.random.default_rng(0)
    dst = np.repeat(np.arange(3000), rng.poisson(150, 3000))
    assert _flushes(dst, 1) == model.flushes(dst, 3000)
    assert model.gnn_atomics(dst, 3000, 300, 152, 2, 1) == 300 * model.flushes(dst, 3000)
    # the carry only removes flushes, more of them with longer runs per warp
    counts = [_flushes(dst, b) for b in (1, 2, 4, 8, 16)]
    assert counts == sorted(counts, reverse=True) and counts[-1] < counts[0] / 2


def test_benchmark_scale_count():
    # the level-1 graph's shape at the benchmark (K = 24 733, E1 = 3.71 M: about 150 edges per destination) gives the
    # 82.9 M atomics of one GNN launch without the carry when every mixed unit runs the segmented scan; the
    # two-destination pass flushes each boundary unit's two destinations once each
    rng = np.random.default_rng(1)
    dst = np.repeat(np.arange(24733), rng.poisson(150, 24733))
    assert abs(model.gnn_atomics(dst, 24733, 300, 152, 2, 1, two_pass=False) / 1e6 - 82.9) < 0.5
    assert model.gnn_atomics(dst, 24733, 300, 152, 2, 1) < 0.95 * model.gnn_atomics(dst, 24733, 300, 152, 2, 1,
                                                                                     two_pass=False)


def test_flush_instructions():
    # car width (152 x 2): a uniform unit issues 5 flush instructions per column group, a mixed one 76
    dst = np.concatenate([np.zeros(40, int), np.ones(24, int)])    # units 0, 1, 3 uniform, unit 2 two destinations
    assert model.flush_instructions(dst, 2, 152, 2, two_pass=False) == (3 * 5 * 2, 76 * 2)
    assert model.flush_instructions(dst, 2, 152, 2) == ((3 + 2) * 5 * 2, 0)
    three = np.concatenate([np.zeros(4, int), np.ones(4, int), np.full(8, 2)])
    assert model.flush_instructions(three, 3, 152, 2) == (0, 76 * 2)
    assert model.flush_instructions(np.zeros(16, int), 1, 128, 1) == (4, 0)


def test_two_destination_units():
    # the destinations of rows 0 and 15, in any order within the unit: one flush each; a third destination, or a row
    # 0 / 15 destination that is neither, sends the unit to the segmented scan
    assert model.flushes(np.tile([0, 1], 8), 2) == 2
    assert model.flushes(np.tile([0, 1], 8), 2, two_pass=False) == 16
    assert model.flushes(np.r_[np.zeros(3, int), np.ones(13, int)], 2) == 2
    assert model.flushes(np.r_[np.zeros(3, int), [2], np.ones(12, int)], 3) == 2 + 2
    # past the end (rows 9 .. 15) and out of range: the valid destination once
    assert model.flushes(np.zeros(9, int), 1) == 1
    assert model.flushes(np.r_[np.zeros(8, int), np.full(8, 7)], 1) == 1

"""The segment max's global atomics per launch, counted, and what a destination carry would leave of them.

    python tools/prof_segmax_carry.py [frames] [reps] [B ...]

Builds the benchmark graphs (frames x 20 000 points, car and ped configs) and counts, with a NumPy model of the
epilogue (pg_tc.cu seg_epilogue) over `dst`, the atomics one segment-max launch issues: the GNN edge layer on the
level-1 graph and the pooling layer's last GEMM on the level-0 graph.  For the GNN layer it also counts a design that
is not built: tiles handed out in blocks of B, each warp owning 16 B contiguous rows of a block and carrying its
destination's maxima in registers from tile to tile (B = 1 is the kernel as it is).  Then times the GNN and pooling
edge layers of the loaded build (PG_LIB_VARIANT=NAME: lab/NAME.so) with tools/prof_edge.py.

The model counts what the epilogue does per 16-row unit (a warp's rows of one tile).  A unit whose 16 rows have one
destination is uniform: reduce-scattered, one flush.  With a carry it flushes only when its warp's next unit has
another destination or is not uniform, or the warp has no next unit.  A unit whose every row has the destination of
its row 0 or of its row 15 is a two-destination unit: one reduce-scattered flush per valid destination of the two,
in launches of one accumulator group (ns = 1; two_pass=False counts the segmented scan that other launches, and the
epilogue before, run on such units).  Any other unit
flushes one run per 8-row half and destination (the segmented scan).  Every flush is one atomic per real output
column of the launch's column group.  flush_instructions() counts the warp-wide flush instructions instead: L3 per
reduce-scattered flush, and one per column pair and half for a unit on the segmented scan, whatever its runs."""
import math
import os
import sys

import numpy as np

GNN_WARPGROUPS = 3   # pg_tc.cu kGnnWarpgroups: the consumer warpgroups of a GNN CTA, 4 warps each


def unit_stats(dst, num_dst, two_pass=True):
    """Per 16-row unit of the edge list: (uniform, its destination, flushes of a unit that is not uniform, whether
    that unit is reduce-scattered).  Rows past the end and out-of-range destinations count as -1 (no flush), as in
    the kernel."""
    dst = np.asarray(dst, dtype=np.int64)
    e = dst.size
    u = (e + 15) // 16
    d = np.full(u * 16, -1, dtype=np.int64)
    d[:e] = np.where((dst >= 0) & (dst < num_dst), dst, -1)
    d = d.reshape(u, 16)
    uniform = (d == d[:, :1]).all(axis=1) & (d[:, 0] >= 0)
    runs = np.zeros(u, dtype=np.int64)
    for h in range(2):
        x = d[:, 8 * h:8 * h + 8]
        head = x >= 0
        head[:, 1:] &= x[:, 1:] != x[:, :-1]
        runs += head.sum(axis=1)
    two = np.zeros(u, dtype=bool)
    if two_pass:
        two = ~uniform & ((d == d[:, :1]) | (d == d[:, 15:])).all(axis=1)
        runs[two] = (d[two, 0] >= 0).astype(np.int64) + ((d[two, 15] >= 0) & (d[two, 15] != d[two, 0]))
    return uniform, d[:, 0], runs, two


def gnn_grid_slots(num_rows, ns, num_sms):
    """CTA slots of a GNN launch (pg_tc.cu launch_wg): each runs GNN_WARPGROUPS warpgroups per column group."""
    num_tiles = (num_rows + 63) // 64
    return min(num_sms // ns, math.ceil(num_tiles / GNN_WARPGROUPS))


def next_unit(num_units, block_tiles, slots):
    """The unit a warp's carry meets next (-1: none).  Block b of B tiles gives warp w the units b 4B + w B + [0, B);
    a warpgroup's next block is GNN_WARPGROUPS x slots blocks on."""
    b4 = 4 * block_tiles
    u = np.arange(num_units, dtype=np.int64)
    t = u % block_tiles
    w = (u % b4) // block_tiles
    nxt = np.where(t < block_tiles - 1, u + 1, (u // b4 + GNN_WARPGROUPS * slots) * b4 + w * block_tiles)
    return np.where(nxt < num_units, nxt, -1)


def flushes(dst, num_dst, block_tiles=1, carry=False, slots=1, two_pass=True):
    """Flushes (one per destination and column) of one column group over the edge list."""
    uniform, d0, runs, _ = unit_stats(dst, num_dst, two_pass)
    mixed = int(runs[~uniform].sum())
    if not carry:
        return int(uniform.sum()) + mixed
    nxt = next_unit(uniform.size, block_tiles, slots)
    has = nxt >= 0
    cont = np.zeros_like(uniform)
    cont[has] = uniform[nxt[has]] & (d0[nxt[has]] == d0[has])
    return int((uniform & ~cont).sum()) + mixed


def group_columns(n, ni, ns):
    """Real output columns of each of a launch's ns column groups of ni."""
    return [max(0, min(ni, n - g * ni)) for g in range(ns)]


def gnn_atomics(dst, num_dst, n, ni, ns, block_tiles=1, num_sms=132, two_pass=True):
    """Global atomics of one GNN edge launch (one CTA per column group) with a carry at block_tiles; block_tiles = 1
    counts the kernel as it is."""
    slots = gnn_grid_slots(len(dst), ns, num_sms)
    f = flushes(dst, num_dst, block_tiles, carry=True, slots=slots, two_pass=two_pass)
    return sum(c * f for c in group_columns(n, ni, ns))


def pool_atomics(dst, num_dst, n, two_pass=True):
    """Global atomics of a pooling (or ROWS) segment-max launch of n real columns: no carry."""
    return n * flushes(dst, num_dst, two_pass=two_pass)


def flush_instructions(dst, num_dst, ni, ns, two_pass=True):
    """(reduce-scattered, segmented-scan) warp-wide flush instructions of one GNN launch without a carry, over all
    column groups: L3 = ceil(ceil(ni / 4, 4) / 8) per group and reduce-scattered flush, ni / 2 per group and unit on the
    segmented scan (each column pair of each 8-row half, with only the run heads' lanes active)."""
    uniform, _, runs, two = unit_stats(dst, num_dst, two_pass)
    l3 = ((ni // 4 + 3) // 4 * 4 // 4 + 1) // 2
    scattered = int(uniform.sum()) + int(runs[two].sum())
    return scattered * l3 * ns, int((~uniform & ~two).sum()) * (ni // 2) * ns


def shape(n):
    """The instruction shape (ni, ns) of an n-wide launch (pg_tc.cu wg_shape)."""
    np_ = (n + 15) // 16 * 16
    for lim, ni, ns in ((64, 64, 1), (128, 128, 1), (192, 96, 2), (256, 128, 2), (304, 152, 2)):
        if np_ <= lim:
            return ni, ns
    raise ValueError(n)


def main():
    import json
    import runpy

    import torch

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    from oracle import synth
    from pointgnn_b200.models import graph_gen

    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 100
    blocks = [int(b) for b in sys.argv[3:]] or [1, 2, 4, 8, 16]
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    fr = [synth.lidar_frame(i, 20000) for i in range(frames)]
    pts = torch.from_numpy(np.vstack([f[0] for f in fr])).cuda()
    fp = torch.arange(frames + 1, dtype=torch.int32, device='cuda') * 20000
    for name in ('car_auto_T3_train', 'ped_cyl_auto_T3_trainval'):
        cfg = json.load(open(os.path.join(root, 'tests/golden/config_%s.json' % name)))
        w = np.load(os.path.join(root, 'tests/golden/weights_%s.npz' % name))
        kw = cfg['runtime_graph_gen_kwargs']
        coords, _, edges = graph_gen.gen_multi_level_local_graph_v3(pts, frame_ptr=fp, **kw)
        k = coords[1].shape[0]   # the level-1 vertices: the pooling layer's keypoints and the GNN's vertices
        d0 = edges[0][:, 1].cpu().numpy()
        d1 = edges[1][:, 1].cpu().numpy()
        gnn_n = int(w['layer2/extract_vertex_features/fully_connected_1/weights'].shape[1])
        s = 'layer1/extract_vertex_features/fully_connected'
        last = max((f for f in w.files if f.startswith(s) and f.endswith('/weights')), key=lambda f: (len(f), f))
        pool_n = int(w[last].shape[1])
        print('%s: E0 %d  E1 %d  K %d  GNN n %d  pooling last n %d  %d SMs' % (name, d0.size, d1.size, k, gnn_n,
                                                                              pool_n, num_sms))
        ni, ns = shape(gnn_n)
        old = gnn_atomics(d1, k, gnn_n, ni, ns, 1, num_sms, two_pass=False)
        print('  GNN edge launch, segmented scan for every mixed unit: %6.1f M atomics' % (old / 1e6))
        base = gnn_atomics(d1, k, gnn_n, ni, ns, 1, num_sms)
        for b in blocks:
            a = gnn_atomics(d1, k, gnn_n, ni, ns, b, num_sms)
            print('  GNN edge launch, B = %2d: %6.1f M atomics (%.2f x B = 1)' % (b, a / 1e6, a / base))
        for tp in (False, True):
            fu, fm = flush_instructions(d1, k, ni, ns, tp)
            print('  GNN edge launch, warp-wide flush instructions%s: %.2f M reduce-scattered, %.2f M segmented scan'
                  % ('' if tp else ' (segmented scan for every mixed unit)', fu / 1e6, fm / 1e6))
        # a last layer wider than one launch runs as several column blocks: every column is flushed once per flush
        # the two-destination pass runs at one accumulator group (ns = 1) only
        pool = pool_atomics(d0, k, pool_n, two_pass=shape(min(pool_n, 304))[1] == 1)
        print('  pooling last GEMM: %6.1f M atomics' % (pool / 1e6))
    sys.argv = [os.path.join(root, 'tools', 'prof_edge.py'), str(frames), str(reps)]
    runpy.run_path(sys.argv[0], run_name='__main__')


if __name__ == '__main__':
    main()

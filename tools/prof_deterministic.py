"""Cost of the ordered segment sum (PG_FLAG_DETERMINISTIC, torch.use_deterministic_algorithms(True)) against the
atomic one, at the benchmark's workloads (car_auto_T3_20k and ped_cyl_auto_T3_20k_b8: 8 frames x 20 000 points,
shipped weights): the GNN edge layer (layer2's edge MLP, level-1 graph) and the pooling layer (layer1's point MLP,
level-0 graph), one prepared-layer call with sum and with mean, switch off and on alternated three times in one
process (best of three), each timed with CUDA events over `reps` calls, at bf16x3 and fp16.  Then pg_scatter_sum over
the level-1 edges with 300 channels, off and on: the on side adds the stable radix sort of the ids.  At car_auto_T3_20k
a torch.profiler run of its own splits one GNN and one pooling call (bf16x3, sum) into kernel times, off and on.
Prints the card and its power limit first.

    python tools/prof_deterministic.py [reps]"""
import json
import os
import re
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import synth  # noqa: E402
from pointgnn_b200 import _lib  # noqa: E402
from pointgnn_b200.models import graph_gen  # noqa: E402

WORKLOADS = {'car_auto_T3_20k': 'car_auto_T3_train', 'ped_cyl_auto_T3_20k_b8': 'ped_cyl_auto_T3_trainval'}
FRAMES, POINTS = 8, 20000


def timed(fn, reps, ordered):
    torch.use_deterministic_algorithms(ordered)
    try:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        a = torch.cuda.Event(enable_timing=True)
        b = torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / reps
    finally:
        torch.use_deterministic_algorithms(False)


def off_on(fn, reps):
    """-> (best ms off, best ms on, max |on - off| / max(1, max |off|))"""
    t = {False: [], True: []}
    for _ in range(3):
        for ordered in (False, True):
            t[ordered].append(timed(fn, reps, ordered))
    off = fn()
    torch.use_deterministic_algorithms(True)
    on = fn()
    torch.use_deterministic_algorithms(False)
    rel = float((on - off).abs().max()) / max(1.0, float(off.abs().max()))
    return min(t[False]), min(t[True]), rel


def breakdown(label, fn, calls=5):
    """GPU time per call by kernel (torch.profiler, CUDA activity, a run of its own), switch off and on."""
    from torch.profiler import ProfilerActivity, profile
    for ordered in (False, True):
        torch.use_deterministic_algorithms(ordered)
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                fn()
            torch.cuda.synchronize()
        torch.use_deterministic_algorithms(False)
        rows = {}
        for ev in prof.key_averages():
            us = getattr(ev, 'self_device_time_total', 0)
            if us > 0:
                name = re.sub(r'^void |[<(].*$', '', ev.key.replace('(anonymous namespace)::', '')).split('::')[-1]
                t, n = rows.get(name, (0.0, 0))
                rows[name] = (t + us / 1e3 / calls, n + ev.count // calls)
        total = sum(t for t, _ in rows.values())
        print('  %s, switch %s: %.3f ms of kernels per call' % (label, 'on' if ordered else 'off', total))
        for name, (t, n) in sorted(rows.items(), key=lambda kv: -kv[1][0]):
            print('    %-40s %3d launches %8.3f ms' % (name[-40:], n, t))


def workload(wl, reps):
    name = WORKLOADS[wl]
    cfg = json.load(open(os.path.join(ROOT, 'tests/golden/config_%s.json' % name)))
    w = dict(np.load(os.path.join(ROOT, 'tests/golden/weights_%s.npz' % name)))
    fr = [synth.lidar_frame(i, POINTS) for i in range(FRAMES)]
    pts = torch.from_numpy(np.vstack([f[0] for f in fr])).cuda()
    inten = torch.from_numpy(np.vstack([f[1] for f in fr])).cuda()
    fp = torch.arange(FRAMES + 1, dtype=torch.int32, device='cuda') * POINTS
    coords, kp, edges = graph_gen.gen_multi_level_local_graph_v3(pts, frame_ptr=fp, **cfg['runtime_graph_gen_kwargs'])
    k = coords[1].shape[0]
    print('\n%s: K %d  E0 %d  E1 %d  reps %d' % (wl, k, edges[0].shape[0], edges[1].shape[0], reps))

    def mlp(scope):
        names = [scope] + [scope + '_%d' % i for i in range(1, 8) if (scope + '_%d/weights' % i) in w]
        return ([torch.from_numpy(w[n + '/weights']).cuda() for n in names],
                [torch.from_numpy(w[n + '/biases']).cuda() for n in names])

    gws, gbs = mlp('layer2/extract_vertex_features/fully_connected')
    gdims = [int(gws[0].shape[0])] + [int(x.shape[1]) for x in gws]
    xyz = coords[1].contiguous()
    src1, dst1 = edges[1][:, 0].contiguous(), edges[1][:, 1].contiguous()
    gen = torch.Generator(device='cuda').manual_seed(0)
    feats = (torch.randn((k, gdims[0] - 3), device='cuda', generator=gen) * 0.3).abs()
    pws, pbs = mlp('layer1/extract_vertex_features/fully_connected')
    pdims = [4] + [int(x.shape[1]) for x in pws]
    src0, dst0 = edges[0][:, 0].contiguous(), edges[0][:, 1].contiguous()
    kpi = kp[0].reshape(-1).contiguous()
    print('%-8s %-6s %-5s %-6s %9s %9s %7s %10s' % ('', '', 'layer', 'agg', 'off ms', 'on ms', 'on/off', 'max rel d'))
    for precision, code in (('bf16x3', 1), ('fp16', 2)):
        g = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_GNN, gws, gbs, gdims, code)
        p = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_POOL, pws, pbs, pdims, code)
        for layer in ('gnn', 'pool'):
            for agg in ('sum', 'mean'):
                if layer == 'gnn':
                    fn = lambda: g.edge_mlp_max(feats, xyz, xyz, None, src1, dst1, k, trusted=True, aggregation=agg)  # noqa: E731,E501
                else:
                    fn = lambda: p.edge_mlp_max(inten, pts, pts, kpi, src0, dst0, k, trusted=True, aggregation=agg)  # noqa: E731,E501
                off, on, rel = off_on(fn, reps)
                print('%-8s %-6s %-5s %-6s %9.3f %9.3f %7.3f %10.2g' % (wl[:8], precision, layer, agg, off, on, on / off,
                                                                     rel))
    if wl == 'car_auto_T3_20k':
        g = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_GNN, gws, gbs, gdims, 1)
        p = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_POOL, pws, pbs, pdims, 1)
        breakdown('gnn bf16x3 sum', lambda: g.edge_mlp_max(feats, xyz, xyz, None, src1, dst1, k, trusted=True,
                                                          aggregation='sum'))
        breakdown('pool bf16x3 sum', lambda: p.edge_mlp_max(inten, pts, pts, kpi, src0, dst0, k, trusted=True,
                                                           aggregation='sum'))
    e = dst1.numel()
    x = torch.randn((e, 300), device='cuda', generator=gen)
    shuffled = dst1[torch.randperm(e, device='cuda', generator=gen)].contiguous()
    for label, ids in (('sorted', dst1), ('shuffled', shuffled)):
        off, on, rel = off_on(lambda: _lib.scatter_sum(x, ids, k), reps)
        print('%-8s pg_scatter_sum [%d, 300], ids %-8s %9.3f %9.3f %7.3f %10.2g' % (wl[:8], e, label, off, on, on / off,
                                                                                   rel))


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print('card: %s (power limit %s)' % tuple((smi[0] if smi else '%s, unknown' % torch.cuda.get_device_name()).split(', ')))
    for wl in WORKLOADS:
        workload(wl, reps)


if __name__ == '__main__':
    main()

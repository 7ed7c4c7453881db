"""Cost of the sum and the mean against the max in the fused edge layers, at the benchmark's workloads
(car_auto_T3_20k and ped_cyl_auto_T3_20k_b8: 8 frames x 20 000 points, shipped weights): the GNN edge layer (layer2's
edge MLP, level-1 graph) and the pooling layer (layer1's point MLP, level-0 graph), each one prepared-layer call timed
with CUDA events, max / sum / mean alternating in one process, at bf16x3 and fp16.  Then, once at car_auto_T3_20k and
bf16x3, GraphNetAutoCenter.apply_regular (layer2) with graph_scatter_sum_fn (fused) against the same sum wrapped in a
user function (the op-by-op route: gather, concat, dense layers over all E edges, scatter), with torch's peak
allocation of each (the library's stream-ordered temporaries, such as the fused route's per-vertex P table, are not in
it).  At ped's E1 = 5.3 M the op-by-op route stops at its first edge layer: K = 303 is not a multiple of 4, so that
layer runs the fp32 dense kernel, whose grid has one row of blocks per 64 edges, more than a launch allows.
Prints the card and its power limit first.

    python tools/prof_aggregation.py [reps]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import synth  # noqa: E402
import pointgnn_b200  # noqa: E402
from pointgnn_b200 import _lib  # noqa: E402
from pointgnn_b200.models import gnn, graph_gen  # noqa: E402

WORKLOADS = {'car_auto_T3_20k': 'car_auto_T3_train', 'ped_cyl_auto_T3_20k_b8': 'ped_cyl_auto_T3_trainval'}
FRAMES, POINTS = 8, 20000


def timed(fn, reps):
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


def peak_gb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 1e9


def user_sum(point_features, point_centers, num_centers):
    """The package's sum behind a function of the user's own: the layer takes the op-by-op route."""
    return gnn.graph_scatter_sum_fn(point_features, point_centers, num_centers)


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
    print('%-8s %-6s %26s %26s' % ('', '', 'GNN edge ms (max/sum/mean)', 'pool edge ms (max/sum/mean)'))
    for precision, code in (('bf16x3', 1), ('fp16', 2)):
        g = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_GNN, gws, gbs, gdims, code)
        p = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_POOL, pws, pbs, pdims, code)
        row = []
        for layer in ('gnn', 'pool'):
            t = {a: [] for a in _lib.AGGREGATIONS}
            for _ in range(3):      # alternate the three, three times each
                for agg in _lib.AGGREGATIONS:
                    if layer == 'gnn':
                        fn = lambda: g.edge_mlp_max(feats, xyz, xyz, None, src1, dst1, k, trusted=True, aggregation=agg)  # noqa: E731,E501
                    else:
                        fn = lambda: p.edge_mlp_max(inten, pts, pts, kpi, src0, dst0, k, trusted=True, aggregation=agg)  # noqa: E731,E501
                    t[agg].append(timed(fn, reps))
            row.append(' / '.join('%6.3f' % min(t[a]) for a in _lib.AGGREGATIONS))
        print('%-8s %-6s %26s %26s' % (wl[:8], precision, row[0], row[1]))
    if wl != 'car_auto_T3_20k':
        return
    # the whole GNN layer, fused against op by op (bf16x3)
    lc = [c for c in cfg['model_kwargs']['layer_configs'] if c['scope'] == 'layer2'][0]
    store = gnn.VariableStore(w)
    pointgnn_b200.set_precision('bf16x3')
    e1 = edges[1].contiguous()

    def layer2(fn):
        def run():
            with gnn.variable_session(store), gnn.variable_scope('layer2'):
                gnn._ctx.trusted_edges = True
                out = gnn.GraphNetAutoCenter(aggregation_fn=fn).apply_regular(feats, xyz, None, e1, **lc['kwargs'])
                gnn._ctx.trusted_edges = False
                return out
        return run

    fused, by_op = layer2(gnn.graph_scatter_sum_fn), layer2(user_sum)
    a, b = fused(), by_op()
    rel = float((a - b).abs().max()) / max(1.0, float(b.abs().max()))
    tf_, tb = timed(fused, max(2, reps // 4)), timed(by_op, 2)
    pf, pb = peak_gb(fused), peak_gb(by_op)
    print('layer2 GraphNetAutoCenter, sum, bf16x3: fused %.3f ms (peak %.2f GB)  op by op %.3f ms (peak %.2f GB)  '
          'x%.1f  max rel diff %.2g' % (tf_, pf, tb, pb, tb / tf_, rel))
    pointgnn_b200.set_precision('fp32')


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print('card: %s (power limit %s)' % tuple((smi[0] if smi else '%s, unknown' % torch.cuda.get_device_name()).split(', ')))
    for wl in WORKLOADS:
        workload(wl, reps)


if __name__ == '__main__':
    main()

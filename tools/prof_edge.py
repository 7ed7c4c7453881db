"""Time the tensor-core layers of one car_auto_T3 forward at the benchmark shape (8 frames x 20 000 points by default):
the prepared GNN edge layer on the level-1 graph, a 300 -> 300 dense layer over its K vertices, and the pooling edge
layer (tools/prof_pool.py).  CUDA events over many launches; prints ms per call and executed TFLOP/s (BF16x3 split,
padded shapes) against the 989 TFLOP/s dense BF16 data-sheet figure of the H100 SXM.

    python tools/prof_edge.py [frames] [reps] [precision]

PG_LIB_VARIANT=NAME runs an experiment build lab/NAME.so (tools/build_variant.sh)."""
import json
import os
import runpy
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import synth  # noqa: E402
from pointgnn_b200 import _lib  # noqa: E402
if os.environ.get('PG_LIB_VARIANT'):
    _lib.LIB_PATH = os.path.join(ROOT, 'lab', os.environ['PG_LIB_VARIANT'] + '.so')
from pointgnn_b200.models import graph_gen  # noqa: E402

PEAK = 989.0     # TFLOP/s, dense BF16, H100 SXM data sheet


def pad16(v):
    return (v + 15) // 16 * 16


def padded_n(n):
    """Output width one tensor-core launch computes for an n-wide layer (instruction shapes 64, 128, 192, 256, 304)."""
    npad = pad16(n)
    for w in (64, 128, 192, 256, 304):
        if npad <= w:
            return w
    raise ValueError('wider than one launch: %d' % n)


def tc_flop(rows, k, n):
    """Executed tensor-core FLOP of a [rows, k] x [k, n] BF16x3 GEMM: three products on the padded shape."""
    return 3 * 2 * rows * pad16(k) * padded_n(n)


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


def report(what, ms, flop):
    tf = flop / ms / 1e9
    print('%-44s %8.3f ms  %6.1f executed TFLOP/s  (%4.1f %% of %g)' % (what, ms, tf, 100 * tf / PEAK, PEAK))


frames = int(sys.argv[1]) if len(sys.argv) > 1 else 8
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
prec = int(sys.argv[3]) if len(sys.argv) > 3 else 1
name = 'car_auto_T3_train'
cfg = json.load(open(os.path.join(ROOT, 'tests/golden/config_%s.json' % name)))
w = dict(np.load(os.path.join(ROOT, 'tests/golden/weights_%s.npz' % name)))
fr = [synth.lidar_frame(i, 20000) for i in range(frames)]
pts = torch.from_numpy(np.vstack([f[0] for f in fr])).cuda()
fp = torch.arange(frames + 1, dtype=torch.int32, device='cuda') * 20000
coords, kp, edges = graph_gen.gen_multi_level_local_graph_v3(pts, frame_ptr=fp, **cfg['runtime_graph_gen_kwargs'])
xyz = coords[1].contiguous()
k = xyz.shape[0]
src, dst = edges[1][:, 0].contiguous(), edges[1][:, 1].contiguous()
e = src.numel()
scope = 'layer2/extract_vertex_features/fully_connected'
ws = [torch.from_numpy(w[scope + s + '/weights']).cuda() for s in ('', '_1')]
bs = [torch.from_numpy(w[scope + s + '/biases']).cuda() for s in ('', '_1')]
dims = [int(ws[0].shape[0])] + [int(x.shape[1]) for x in ws]
c = dims[0] - 3
gen = torch.Generator(device='cuda').manual_seed(0)
feats = (torch.randn((k, c), device='cuda', generator=gen) * 0.3).abs()     # level-1 vertex features, ReLU-like
print('frames %d  K %d  E1 %d  precision %d  edge MLP %s' % (frames, k, e, prec, 'x'.join(map(str, dims))))

edge = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_GNN, ws, bs, dims, prec)
ms = timed(lambda: edge.edge_mlp_max(feats, xyz, xyz, None, src, dst, k, trusted=True), reps)
# the hoisted per-vertex table P = F @ W1[:C] + b1, then the per-edge second layer
report('GNN edge layer (P GEMM + fill + fused kernel)', ms, tc_flop(k, c, dims[1]) + tc_flop(e, dims[1], dims[2]))

wd = torch.from_numpy(w['layer2/combined_features/fully_connected/weights']).cuda()
bd = torch.from_numpy(w['layer2/combined_features/fully_connected/biases']).cuda()
dense = _lib.PreparedLayer(_lib.PG_LAYER_MLP, [wd], [bd], [int(wd.shape[0]), int(wd.shape[1])], prec)
x = torch.randn((k, int(wd.shape[0])), device='cuda', generator=gen)
ms = timed(lambda: dense.mlp(x, last_linear=False), reps)
report('dense %dx%d over the K vertices' % tuple(wd.shape), ms, tc_flop(k, *wd.shape))

sys.argv = [os.path.join(ROOT, 'tools', 'prof_pool.py'), str(frames), str(reps), str(prec)]
pool = runpy.run_path(sys.argv[0], run_name='__main__')
pdims, e0 = pool['dims'], pool['src'].numel()
# layer 0 runs in fp32 inside the producer of layer 1; layers 1 .. L-1 are tensor-core GEMMs over the edges
report('pooling edge layer (%s)' % 'x'.join(map(str, pdims)), pool['ms'],
       sum(tc_flop(e0, pdims[i], pdims[i + 1]) for i in range(1, len(pdims) - 1)))

"""Drive only the pooling-layer kernel (PointSetPooling edge part) for ncu / timing."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import synth  # noqa: E402
from pointgnn_b200 import _lib  # noqa: E402
if os.environ.get('PG_LIB_VARIANT'):      # experiment builds (tools/build_variant.sh NAME -DFLAG...): lab/<NAME>.so
    _lib.LIB_PATH = os.path.join(ROOT, 'lab', os.environ['PG_LIB_VARIANT'] + '.so')
from pointgnn_b200.models import graph_gen  # noqa: E402

frames = int(sys.argv[1]) if len(sys.argv) > 1 else 8
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
prec = int(sys.argv[3]) if len(sys.argv) > 3 else 1
name = sys.argv[4] if len(sys.argv) > 4 else 'car_auto_T3_train'       # or ped_cyl_auto_T3_trainval (last layer 256 -> 512 in two column blocks)
cfg = json.load(open(os.path.join(ROOT, 'tests/golden/config_%s.json' % name)))
w = dict(np.load(os.path.join(ROOT, 'tests/golden/weights_%s.npz' % name)))
fr = [synth.lidar_frame(i, 20000) for i in range(frames)]
pts = torch.from_numpy(np.vstack([f[0] for f in fr])).cuda()
inten = torch.from_numpy(np.vstack([f[1] for f in fr])).cuda()
fp = torch.arange(frames + 1, dtype=torch.int32, device='cuda') * 20000
coords, kp, edges = graph_gen.gen_multi_level_local_graph_v3(pts, frame_ptr=fp, **cfg['runtime_graph_gen_kwargs'])
k = coords[1].shape[0]
s = 'layer1/extract_vertex_features/fully_connected'
names = [s] + [s + '_%d' % i for i in range(1, 8) if (s + '_%d/weights' % i) in w]
ws = [torch.from_numpy(w[n + '/weights']).cuda() for n in names]
bs = [torch.from_numpy(w[n + '/biases']).cuda() for n in names]
src, dst = edges[0][:, 0].contiguous(), edges[0][:, 1].contiguous()
kpi = kp[0].reshape(-1).contiguous()
print('K', k, 'E0', src.numel())
dims = [4] + [int(x.shape[1]) for x in ws]
layer = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_POOL, ws, bs, dims, prec)     # weights packed once, as the model does
flop_per_edge = sum(2 * dims[i] * dims[i + 1] for i in range(len(dims) - 1))
if prec == 1:
    ref = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_POOL, ws, bs, dims, 0).edge_mlp_max(inten, pts, pts, kpi, src, dst, k, trusted=True)
    got = layer.edge_mlp_max(inten, pts, pts, kpi, src, dst, k, trusted=True)
    print('max |tensor-core - fp32 FFMA| = %.3g (empty segments equal: %s)' % (
        float((got - ref).abs()[ref > -1e30].max()), bool(((got < -1e30) == (ref < -1e30)).all())))
for _ in range(2):
    layer.edge_mlp_max(inten, pts, pts, kpi, src, dst, k, trusted=True)
torch.cuda.synchronize()
a = torch.cuda.Event(enable_timing=True)
b = torch.cuda.Event(enable_timing=True)
a.record()
for _ in range(reps):
    layer.edge_mlp_max(inten, pts, pts, kpi, src, dst, k, trusted=True)
b.record()
b.synchronize()
ms = a.elapsed_time(b) / reps
print('pool edge_mlp_max (prepared layer, %s) precision %d: %.3f ms per call, %.1f algorithmic TFLOP/s'
      % ('x'.join(str(d) for d in dims), prec, ms, src.numel() * flop_per_edge / ms / 1e9))

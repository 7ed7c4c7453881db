"""Cost of the activations other than ReLU at the benchmark shape (8 frames x 20 000 points, car_auto_T3 weights):
the GNN edge layer, the pooling edge layer and the whole GNN forward (graph given), each timed with CUDA events for
every activation, alternating with ReLU in the same process.  Prints the card and its power limit first.

    python tools/prof_activation.py [frames] [reps] [precision]"""
import copy
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
from pointgnn_b200.models import gnn, graph_gen, models  # noqa: E402

OTHERS = ['NONE', 'ReLU6', 'LeakyReLU', 'ELU', 'Sigmoid', 'Tanh']
KEYS = ('point_MLP_activation_type', 'output_MLP_activation_type', 'edge_MLP_activation_type',
        'update_MLP_activation_type', 'auto_offset_MLP_feature_activation_type', 'activation_type')


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


def main():
    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    precision = sys.argv[3] if len(sys.argv) > 3 else 'bf16x3'
    prec = 1 if precision == 'bf16x3' else 0
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print('card: %s (power limit %s)' % tuple((smi[0] if smi else '%s, unknown' % torch.cuda.get_device_name()).split(', ')))
    name = 'car_auto_T3_train'
    cfg = json.load(open(os.path.join(ROOT, 'tests/golden/config_%s.json' % name)))
    w = dict(np.load(os.path.join(ROOT, 'tests/golden/weights_%s.npz' % name)))
    fr = [synth.lidar_frame(i, 20000) for i in range(frames)]
    pts = torch.from_numpy(np.vstack([f[0] for f in fr])).cuda()
    inten = torch.from_numpy(np.vstack([f[1] for f in fr])).cuda()
    fp = torch.arange(frames + 1, dtype=torch.int32, device='cuda') * 20000
    coords, kp, edges = graph_gen.gen_multi_level_local_graph_v3(pts, frame_ptr=fp, **cfg['runtime_graph_gen_kwargs'])
    k = coords[1].shape[0]
    print('frames %d  K %d  E0 %d  E1 %d  precision %s  reps %d' % (frames, k, edges[0].shape[0], edges[1].shape[0],
                                                                    precision, reps))

    def mlp(scope):
        names = [scope] + [scope + '_%d' % i for i in range(1, 8) if (scope + '_%d/weights' % i) in w]
        return ([torch.from_numpy(w[n + '/weights']).cuda() for n in names],
                [torch.from_numpy(w[n + '/biases']).cuda() for n in names])

    # GNN edge layer: level-1 graph, layer2's edge MLP, ReLU-like vertex features
    gws, gbs = mlp('layer2/extract_vertex_features/fully_connected')
    gdims = [int(gws[0].shape[0])] + [int(x.shape[1]) for x in gws]
    xyz = coords[1].contiguous()
    src1, dst1 = edges[1][:, 0].contiguous(), edges[1][:, 1].contiguous()
    gen = torch.Generator(device='cuda').manual_seed(0)
    feats = (torch.randn((k, gdims[0] - 3), device='cuda', generator=gen) * 0.3).abs()
    # pooling edge layer: level-0 graph, layer1's point MLP
    pws, pbs = mlp('layer1/extract_vertex_features/fully_connected')
    pdims = [4] + [int(x.shape[1]) for x in pws]
    src0, dst0 = edges[0][:, 0].contiguous(), edges[0][:, 1].contiguous()
    kpi = kp[0].reshape(-1).contiguous()

    def layers(act):
        code = gnn.activation_fn_dict[act]
        g = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_GNN, gws, gbs, gdims, prec, code)
        p = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_POOL, pws, pbs, pdims, prec, code)
        return (lambda: g.edge_mlp_max(feats, xyz, xyz, None, src1, dst1, k, trusted=True),
                lambda: p.edge_mlp_max(inten, pts, pts, kpi, src0, dst0, k, trusted=True))

    def model(act):
        lcs = copy.deepcopy(cfg['model_kwargs']['layer_configs'])
        for lc in lcs:
            for key in KEYS:
                if key in lc['kwargs']:
                    lc['kwargs'][key] = act
        m = models.get_model(cfg['model_name'])(num_classes=cfg['num_classes'], box_encoding_len=7, mode='test',
                                                **dict(cfg['model_kwargs'], layer_configs=lcs))
        m.load_weights(w)
        return lambda: m.predict(inten, coords, kp, edges, is_training=True)

    pointgnn_b200.set_precision(precision)
    relu_layers, relu_model = layers('ReLU'), model('ReLU')
    print('%-10s %14s %14s %14s   (ReLU measured right before each row)' % ('activation', 'GNN edge ms', 'pool edge ms',
                                                                             'forward ms'))
    for act in OTHERS:
        other_layers, other_model = layers(act), model(act)
        row = []
        for fn_relu, fn_other in ((relu_layers[0], other_layers[0]), (relu_layers[1], other_layers[1]),
                                  (relu_model, other_model)):
            row.append((timed(fn_relu, reps), timed(fn_other, reps)))
        print('%-10s %s' % (act, ' '.join('%6.3f / %6.3f' % (r, o) for r, o in row)))


if __name__ == '__main__':
    main()

"""BF16x3 against FP16 on the benchmark workloads: device-timed frames/s, the GNN edge layer and the pooling edge
layer per call, and how far FP16's logits and boxes are from BF16x3's on the same frames.

Each workload (``car_auto_T3_20k``, ``ped_cyl_auto_T3_20k_b8``) is built the way bench.py builds it (its config,
weights, frame seeds and frames per step; L2 flushed between timed steps, CUDA events around graph build + forward
pass + softmax).  The two arithmetics run alternately, REPEATS runs each, after one untimed warm-up of each; the
edge layers are timed as bench.py times the GNN edge kernel (CUDA events around 5 calls of a prepared layer on one
step's graph, after 2 warm-up calls).  Prints one JSON line per run, one summary line per (workload, arithmetic)
with the median of the runs, and the GPU's name, power limit and SM clocks read in the same process.

    python tools/prof_precision.py [--steps 24] [--repeats 3] [--workloads car_auto_T3_20k ped_cyl_auto_T3_20k_b8]
                                   [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (WORKLOADS, load_config, time_edge_kernel: the benchmark's own definitions)

ARITHMETICS = ('bf16x3', 'fp16')


def gpu_conditions():
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True)
    return out.stdout.strip() if out.returncode == 0 else 'unknown (nvidia-smi failed)'


def time_pool_kernel(model, graph_fn, gkw, dev_step, config):
    """CUDA-event ms per call of the pooling edge layer (point MLP + segment max) on one step's graph."""
    import torch
    import pointgnn_b200
    from pointgnn_b200 import _lib
    from pointgnn_b200.models import gnn
    xyz, inten, fp = dev_step
    coords, kp, edges = graph_fn(xyz, frame_ptr=fp, **gkw)
    lc = [l for l in config['model_kwargs']['layer_configs'] if l['type'] == 'scatter_max_point_set_pooling'][0]
    d = lc['kwargs']['point_MLP_depth_list']
    with gnn.variable_session(model._store), gnn.variable_scope(lc['scope']), \
            gnn.variable_scope('extract_vertex_features'):
        ws, bs = gnn._take_mlp_weights(len(d))
    layer = _lib.PreparedLayer(_lib.PG_LAYER_EDGE_POOL, ws, bs, [inten.shape[1] + 3] + list(d),
                               pointgnn_b200.get_precision())
    src, dst = edges[0][:, 0].contiguous(), edges[0][:, 1].contiguous()
    kpi = kp[0].reshape(-1).to(torch.int32).contiguous()
    args = (inten.contiguous(), coords[0], coords[0], kpi, src, dst, kpi.numel())
    for _ in range(2):
        layer.edge_mlp_max(*args, trusted=True)
    torch.cuda.synchronize()
    reps = 5
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        layer.edge_mlp_max(*args, trusted=True)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--steps', type=int, default=24)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--workloads', nargs='+', default=['car_auto_T3_20k', 'ped_cyl_auto_T3_20k_b8'])
    ap.add_argument('--out', default='', help='also write the JSON lines to this file')
    args = ap.parse_args()
    import torch
    import pointgnn_b200
    from oracle import synth
    from pointgnn_b200 import _lib
    from pointgnn_b200.models import graph_gen, models
    from pointgnn_b200.utils import sharding
    assert torch.cuda.is_available() and _lib.tc_available(), 'needs an sm_90 GPU'
    dev = torch.device('cuda', 0)
    lines = []

    def emit(line):
        print(json.dumps(line), flush=True)
        lines.append(line)

    for wl in args.workloads:
        cfg_name, num_points, full_360, fps = bench.WORKLOADS[wl]
        config, weights = bench.load_config(cfg_name)
        graph_fn = graph_gen.get_graph_generate_fn(config['graph_gen_method'])
        gkw = config['runtime_graph_gen_kwargs']
        pool = min(args.steps, bench.FRAME_POOL)
        steps = []
        for s in range(pool):
            pts, inten = [], []
            for f in range(fps):
                x, it = synth.lidar_frame(sharding.frame_seed(s, f, 0, fps), num_points, full_360)
                pts.append(x)
                inten.append(it)
            fp = torch.from_numpy(np.arange(fps + 1, dtype=np.int32) * num_points).to(dev)
            steps.append((torch.from_numpy(np.vstack(pts)).to(dev), torch.from_numpy(np.vstack(inten)).to(dev), fp))
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        mdl = {}
        for arith in ARITHMETICS:
            pointgnn_b200.set_precision(arith)
            mdl[arith] = models.get_model(config['model_name'])(num_classes=config['num_classes'], box_encoding_len=7,
                                                                mode='test', **config['model_kwargs'])
            mdl[arith].load_weights(weights)

        def run(arith):
            """frames/s over args.steps steps, and each pool step's (logits, boxes) on the host."""
            pointgnn_b200.set_precision(arith)
            model = mdl[arith]
            ms, outs = 0.0, {}
            for s in range(args.steps):
                xyz, inten, fp = steps[s % pool]
                flush.zero_()
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                coords, kp, edges = graph_fn(xyz, frame_ptr=fp, **gkw)
                logits, boxes = model.predict(inten, coords, kp, edges, is_training=True)
                model.postprocess(logits)
                b.record()
                b.synchronize()
                ms += a.elapsed_time(b)
                if s < pool:
                    outs[s] = (logits.cpu().numpy(), boxes.cpu().numpy())
            return args.steps * fps / (ms * 1e-3), outs

        for arith in ARITHMETICS:
            run(arith)
        runs = {a: [] for a in ARITHMETICS}
        outs = {}
        for rep in range(args.repeats):
            for arith in ARITHMETICS:
                fps_value, outs[arith] = run(arith)
                runs[arith].append(fps_value)
                emit({'workload': wl, 'precision': arith, 'repeat': rep, 'frames_per_s': fps_value})
        kernels = {}
        for arith in ARITHMETICS:
            pointgnn_b200.set_precision(arith)
            edge_ms, _, reps = bench.time_edge_kernel(mdl[arith], graph_fn, gkw, steps[0], config)
            kernels[arith] = (edge_ms / reps, time_pool_kernel(mdl[arith], graph_fn, gkw, steps[0], config))
        pointgnn_b200.set_precision('fp32')
        for arith in ARITHMETICS:
            dl = max(float(np.abs(outs[arith][s][0] - outs['bf16x3'][s][0]).max()) for s in outs[arith])
            db = max(float(np.abs(outs[arith][s][1] - outs['bf16x3'][s][1]).max()) for s in outs[arith])
            emit({'workload': wl, 'precision': arith, 'summary': True, 'runs': len(runs[arith]),
                  'frames_per_s_median': float(np.median(runs[arith])), 'frames_per_s_min': min(runs[arith]),
                  'frames_per_s_max': max(runs[arith]), 'gnn_edge_layer_ms': kernels[arith][0],
                  'pool_edge_layer_ms': kernels[arith][1], 'max_abs_dlogit_vs_bf16x3': dl,
                  'max_abs_dbox_vs_bf16x3': db, 'frames_compared': pool * fps})
        del flush, steps, mdl
        torch.cuda.empty_cache()
    emit({'gpu': gpu_conditions()})
    if args.out:
        with open(args.out, 'w') as f:
            for line in lines:
                f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
    main()

"""CPU emulation of tensor-core operand roundings on the real checkpoints: max |logit / box error| vs the
fp32 oracle for each candidate arithmetic of the wide (K >= 32) fully-connected layers.  Evidence for DESIGN.md
(why BF16x3 and not a single fp16 / tf32 / bf16 pass).  Test infrastructure: imports oracle/."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle import gnn as ognn  # noqa: E402
from conftest import load_golden  # noqa: E402


def rnd(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dt).to(torch.float32).numpy().astype(np.float64)


def tf32(a):
    b = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    b = ((b + 0x1000) & 0xFFFFE000).astype(np.uint32)    # round-to-nearest (ties away) to 10 mantissa bits
    return b.view(np.float32).astype(np.float64)


def split(a, dt):
    hi = rnd(a, dt)
    lo = rnd(np.asarray(a, dtype=np.float64) - hi, dt)
    return hi, lo


def make_dense(mode):
    def _dense(x, w, b, act, tc=False):
        if mode == 'fp32' or w.shape[0] < 32:
            y = x @ w.astype(x.dtype) + b.astype(x.dtype)[None, :]
        else:
            if mode == 'bf16x1':
                y = rnd(x, torch.bfloat16) @ rnd(w, torch.bfloat16)
            elif mode == 'fp16x1':
                y = rnd(x, torch.float16) @ rnd(w, torch.float16)
            elif mode == 'tf32x1':
                y = tf32(x) @ tf32(w)
            elif mode == 'fp16x2a':      # A split in two fp16, W single fp16
                h, l = split(x, torch.float16)
                wh = rnd(w, torch.float16)
                y = h @ wh + l @ wh
            elif mode == 'bf16x3':
                h, l = split(x, torch.bfloat16)
                wh, wl = split(w, torch.bfloat16)
                y = h @ wh + l @ wh + h @ wl
            elif mode == 'fp16x3':
                h, l = split(x, torch.float16)
                wh, wl = split(w, torch.float16)
                y = h @ wh + l @ wh + h @ wl
            else:
                raise KeyError(mode)
            y = (y + b.astype(np.float64)[None, :]).astype(np.float32)
        return ognn.activate(act, y)
    return _dense


def main():
    orig = ognn._dense
    for name in ('car_auto_T3_train', 'ped_cyl_auto_T3_trainval'):
        g = load_golden(name)
        coords, kp, edges = g.graph_tuple()
        inten = g.graph['intensity']
        args = (g.weights, g.layer_configs, g.config['num_classes'], 7, inten, coords, kp, edges)
        ognn._dense = orig
        l64, b64 = ognn.predict(*args, dtype=np.float64)
        l32, b32 = ognn.predict(*args)
        print('%s: |logit| max %.2f, |box| max %.2f; fp32 vs fp64: %.2e / %.2e' % (
            name, np.abs(l32).max(), np.abs(b32).max(), np.abs(l32 - l64).max(), np.abs(b32 - b64).max()))
        for mode in ('bf16x3', 'fp16x3', 'fp16x2a', 'fp16x1', 'tf32x1', 'bf16x1'):
            ognn._dense = make_dense(mode)
            l, b = ognn.predict(*args)
            print('   %-8s max|dlogit| %.2e  max|dbox| %.2e   (vs fp32 oracle)' % (
                mode, np.abs(l - l32).max(), np.abs(b - b32).max()))
    ognn._dense = orig


if __name__ == '__main__':
    main()

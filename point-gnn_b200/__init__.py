"""point-gnn_b200: H100 (sm_90a) implementation of Point-GNN's per-frame message-passing path.

Host side = a Python mirror of the reference's own layer / op API
(``models.graph_gen``, ``models.gnn``, ``models.models``); compute side =
hand-written sm_90a CUDA kernels in ``libpointgnn_b200.so`` behind the C ABI of
``include/pointgnn_b200.h``.  There is no CPU fallback: importing the op layer
without the built library raises.
"""
__version__ = '0.1.0'

PRECISION_FP32 = 0      # fp32 FFMA kernels (bit-faithful association order)
PRECISION_BF16X3 = 1    # Hopper wgmma tensor cores, 3-term BF16 split (fp32-class accuracy)
PRECISION_FP16 = 2      # Hopper wgmma tensor cores, operands rounded once to FP16, fp32 accumulation (opt-in)

_precision = PRECISION_FP32


def set_precision(precision):
    """Select the arithmetic of the dense layers: 'fp32', 'bf16x3' or 'fp16' (both wgmma)."""
    global _precision
    table = {'fp32': PRECISION_FP32, 'bf16x3': PRECISION_BF16X3, 'fp16': PRECISION_FP16,
             PRECISION_FP32: PRECISION_FP32, PRECISION_BF16X3: PRECISION_BF16X3, PRECISION_FP16: PRECISION_FP16}
    if precision not in table:
        raise ValueError('unknown precision %r' % (precision,))
    _precision = table[precision]


def get_precision():
    return _precision

"""The FP16 precision (code 2) without a GPU: the FP16 oracle against the fp32 goldens and the Python and run.py
plumbing.  The compile-time checks of the FP16 tensor-core instances are in test_tc_build_cpu.py."""
import tempfile

import numpy as np
import pytest

from conftest import ALL_CHECKPOINTS, load_golden
from oracle import gnn as ognn

LOGIT_TOL, BOX_TOL = 2e-2, 1e-2


@pytest.mark.parametrize('name', ALL_CHECKPOINTS)
def test_oracle_within_bounds_of_fp32_golden(name):
    """The FP16 arithmetic of every shipped checkpoint stays within the bounds the GPU tests hold the kernels to."""
    g = load_golden(name)
    coords, kp, edges = g.graph_tuple()
    logits, boxes = ognn.predict(g.weights, g.layer_configs, g.config['num_classes'], 7, g.graph['intensity'], coords,
                                 kp, edges, fp16=True)
    assert logits.shape == g.gnn['logits'].shape and boxes.shape == g.gnn['boxes'].shape
    dl, db = np.abs(logits - g.gnn['logits']).max(), np.abs(boxes - g.gnn['boxes']).max()
    assert dl <= LOGIT_TOL and db <= BOX_TOL, (name, dl, db)
    # and it really rounds: FP16 is far from the fp32 answer at the 1e-4 scale BF16x3 reaches
    assert dl > 1e-4, (name, dl)


def test_oracle_rounding():
    x = np.array([[1.0 + 2.0 ** -12, 70000.0, -1e9, 3.0]], np.float32)
    r = ognn.f16(x)
    assert r[0, 0] == 1.0 and r[0, 1] == 65504.0 and r[0, 2] == -65504.0 and r[0, 3] == 3.0
    # exact products and sums of the rounded operands, rounded once to fp32
    w = np.full((4, 1), 1.0, np.float32)
    assert ognn.tc_gemm(x, w)[0, 0] == np.float32(1.0 + 65504.0 - 65504.0 + 3.0)
    assert ognn.fc_uses_tc(300, 64) and not ognn.fc_uses_tc(64, 7) and not ognn.fc_uses_tc(32, 64)
    # the car GNN layer (303 -> 300 -> 300): W resident in 152-wide column groups, 92 KB of FP16 each
    assert ognn.gnn_uses_tc([303, 300, 300]) and not ognn.gnn_uses_tc([303, 300, 300, 300])
    assert ognn.pool_uses_tc([4, 32, 64, 128, 300], 'ReLU')
    assert not ognn.pool_uses_tc([4, 32, 64, 128, 300], 'Tanh')


def test_set_precision_fp16():
    import pointgnn_b200
    prev = pointgnn_b200.get_precision()
    try:
        pointgnn_b200.set_precision('fp16')
        assert pointgnn_b200.get_precision() == pointgnn_b200.PRECISION_FP16 == 2
        pointgnn_b200.set_precision(pointgnn_b200.PRECISION_FP16)
        assert pointgnn_b200.get_precision() == 2
        with pytest.raises(ValueError):
            pointgnn_b200.set_precision('fp8')
        with pytest.raises(ValueError):
            pointgnn_b200.set_precision(3)
    finally:
        pointgnn_b200.set_precision(prev)


def test_run_parses_precision_fp16():
    from pointgnn_b200 import run
    with tempfile.TemporaryDirectory() as d:
        # the arguments parse; the checkpoint directory has no config, which is the first thing main() checks
        with pytest.raises(AssertionError, match='No config file'):
            run.main([d, '--precision', 'fp16'])
        with pytest.raises(SystemExit):
            run.main([d, '--precision', 'fp8'])

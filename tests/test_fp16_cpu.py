"""The FP16 precision (code 2) without a GPU: the FP16 oracle against the fp32 goldens, the Python and run.py
plumbing, and compile-time checks of the FP16 tensor-core instances.  pg_tc.cu built with the Makefile's flags must
give every FP16 instance (wg_gemm_f16_kernel, wg_gemm_act_f16_kernel) wgmmas that ptxas does not serialise, no
spills, and the GNN edge layer's FP16 instances must build A in registers (no shared-memory A store, no warpgroup
barrier) and issue F16 HGMMAs only."""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import fp16_oracle
from conftest import ALL_CHECKPOINTS, load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'point-gnn_b200', 'csrc')
F16_KERNELS = ('wg_gemm_f16_kernel', 'wg_gemm_act_f16_kernel')
LOGIT_TOL, BOX_TOL = 2e-2, 1e-2


@pytest.mark.parametrize('name', ALL_CHECKPOINTS)
def test_oracle_within_bounds_of_fp32_golden(name):
    """The FP16 arithmetic of every shipped checkpoint stays within the bounds the GPU tests hold the kernels to."""
    g = load_golden(name)
    coords, kp, edges = g.graph_tuple()
    logits, boxes = fp16_oracle.predict(g.weights, g.layer_configs, g.config['num_classes'], 7, g.graph['intensity'],
                                        coords, kp, edges)
    assert logits.shape == g.gnn['logits'].shape and boxes.shape == g.gnn['boxes'].shape
    dl, db = np.abs(logits - g.gnn['logits']).max(), np.abs(boxes - g.gnn['boxes']).max()
    assert dl <= LOGIT_TOL and db <= BOX_TOL, (name, dl, db)
    # and it really rounds: FP16 is far from the fp32 answer at the 1e-4 scale BF16x3 reaches
    assert dl > 1e-4, (name, dl)


def test_oracle_rounding():
    x = np.array([[1.0 + 2.0 ** -12, 70000.0, -1e9, 3.0]], np.float32)
    r = fp16_oracle.f16(x)
    assert r[0, 0] == 1.0 and r[0, 1] == 65504.0 and r[0, 2] == -65504.0 and r[0, 3] == 3.0
    # exact products and sums of the rounded operands, rounded once to fp32
    w = np.full((4, 1), 1.0, np.float32)
    assert fp16_oracle.tc_gemm(x, w)[0, 0] == np.float32(1.0 + 65504.0 - 65504.0 + 3.0)
    assert fp16_oracle.fc_uses_tc(300, 64) and not fp16_oracle.fc_uses_tc(64, 7) and not fp16_oracle.fc_uses_tc(32, 64)
    # the car GNN layer (303 -> 300 -> 300): W resident in 152-wide column groups, 92 KB of FP16 each
    assert fp16_oracle.gnn_uses_tc([303, 300, 300]) and not fp16_oracle.gnn_uses_tc([303, 300, 300, 300])
    assert fp16_oracle.pool_uses_tc([4, 32, 64, 128, 300], 'ReLU')
    assert not fp16_oracle.pool_uses_tc([4, 32, 64, 128, 300], 'Tanh')


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


# ---- compile-time checks of the FP16 instances ------------------------------------------------------------------
def _make_var(name):
    # the Makefile's own value of a variable (an extra makefile on stdin prints it)
    out = subprocess.run(['make', '--no-print-directory', '-s', '-C', CSRC, '-f', 'Makefile', '-f', '-', 'print-var'],
                         input='print-var:\n\t@echo $(%s)\n' % name, capture_output=True, text=True, check=True)
    return out.stdout.strip()


@pytest.fixture(scope='module')
def build(tmp_path_factory):
    """(ptxas log, SASS per function name) of pg_tc.cu compiled with the Makefile's flags."""
    if shutil.which('make') is None:
        pytest.skip('make not found')
    nvcc = _make_var('NVCC')
    nvcc = nvcc if os.path.isfile(nvcc) else shutil.which(nvcc)
    if not nvcc:
        pytest.skip('nvcc not found')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    if not os.path.isfile(cuobjdump):
        pytest.skip('cuobjdump not found next to nvcc')
    flags = _make_var('NVCCFLAGS').split()
    assert '-v' in flags and 'arch=compute_90a,code=sm_90a' in flags
    obj = str(tmp_path_factory.mktemp('f16') / 'pg_tc.o')
    res = subprocess.run([nvcc] + flags + ['-c', 'pg_tc.cu', '-o', obj], cwd=CSRC, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log[-4000:]
    sass = subprocess.run([cuobjdump, '-sass', obj], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r'\n\s*Function : ', sass)[1:]:
        name, _, body = part.partition('\n')
        funcs[name.strip()] = body
    return log, funcs


def _is_f16(name):
    return any(k in name for k in F16_KERNELS)


def test_fp16_instances_not_serialised_and_no_spills(build):
    log, _ = build
    # C7518: wgmmas serialised for a reason in the code; C7512: for want of registers
    serialised = [m for m in re.findall(r'\(C75(?:18|12)\)[^\n]*\'(\S+)\'', log) if _is_f16(m)]
    assert not serialised, 'ptxas serialises the wgmmas of %d FP16 instances, e.g. %s' % (len(serialised), serialised[0])
    props = re.findall(r'Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                       r'(\d+) bytes spill loads', log)
    f16 = [p for p in props if 'wg_gemm_f16_kernel' in p[0]]
    act = [p for p in props if 'wg_gemm_act_f16_kernel' in p[0]]
    # as wg_gemm_kernel: 3 producers x 2 epilogues, minus GNN with the store epilogue, x 5 instruction shapes; the
    # any-activation GNN instances x 5 shapes
    assert len(f16) == 25 and len(act) == 5, ([p[0] for p in f16], [p[0] for p in act])
    spilled = [p for p in f16 + act if p[2] != '0' or p[3] != '0']
    assert not spilled, 'spills in %s' % [(p[0], p[2], p[3]) for p in spilled]


def test_fp16_gnn_edge_layer_takes_a_from_registers(build):
    _, funcs = build
    # kProd is the first template argument; PROD_GNN = 1
    gnn = {n: b for n, b in funcs.items() if any(re.search(k + r'ILi1ELi', n) for k in F16_KERNELS)}
    assert len(gnn) == 10, sorted(gnn)
    for name, body in gnn.items():
        hgmma = re.findall(r'HGMMA\.\S+\s+([^;]*);', body)
        assert hgmma, name
        ss = [h for h in hgmma if not re.match(r'R\d+, R\d+, gdesc\[', h)]
        assert not ss, '%s: %d of %d HGMMAs read A from shared memory, e.g. %s' % (name, len(ss), len(hgmma), ss[0])
        sts = re.findall(r'\bSTS(?:\.\S+)?\s[^;]*;', body)
        assert not sts, '%s stores to shared memory: %s' % (name, sts[:4])
        counted = re.findall(r'\bBAR\.SYNC\S*\s+[^;,]+,[^;]*;', body)
        assert not counted, '%s syncs a warpgroup: %s' % (name, counted)


def test_fp16_instances_issue_f16_hgmmas_only(build):
    _, funcs = build
    # the SASS of an HGMMA names its input type after the accumulator's, except FP16, the default:
    # "HGMMA.64x152x16.F32 ..." is FP16, "HGMMA.64x152x16.F32.BF16 ..." BF16
    def kinds(body):
        return [k or 'F16' for k in re.findall(r'HGMMA\.\d+x\d+x16\.F32(?:\.(\w+))?\s', body)]
    f16 = {n: b for n, b in funcs.items() if _is_f16(n)}
    assert len(f16) == 30, sorted(f16)
    n_f16 = 0
    for name, body in f16.items():
        k = kinds(body)
        assert k and set(k) == {'F16'}, (name, sorted(set(k)))
        n_f16 += len(k)
    # the BF16x3 instances stay BF16, with three HGMMAs for every FP16 one
    bf16 = [kinds(b) for n, b in funcs.items() if 'wg_gemm_kernel' in n or 'wg_gemm_act_kernel' in n]
    assert all(k and set(k) == {'BF16'} for k in bf16)
    assert sum(len(k) for k in bf16) == 3 * n_f16

"""Compile-time checks of the register-A (RS) wgmma path of the tensor-core kernel (no GPU needed).  pg_tc.cu built
with the Makefile's nvcc flags must not let ptxas serialise the wgmmas of any wg_gemm_kernel / wg_gemm_act_kernel
instance, for any reason, and the GNN edge layer's instances must build A in registers: every HGMMA takes A from a
register, and the kernel neither stores A to shared memory nor syncs a warpgroup per chunk."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'point-gnn_b200', 'csrc')
KERNELS = ('wg_gemm_kernel', 'wg_gemm_act_kernel')


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
    obj = str(tmp_path_factory.mktemp('rs') / 'pg_tc.o')
    res = subprocess.run([nvcc] + flags + ['-c', 'pg_tc.cu', '-o', obj], cwd=CSRC, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log[-4000:]
    sass = subprocess.run([cuobjdump, '-sass', obj], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r'\n\s*Function : ', sass)[1:]:
        name, _, body = part.partition('\n')
        funcs[name.strip()] = body
    return log, funcs


def _is_gnn(name):
    # kProd is the first template argument; PROD_GNN = 1
    return any(re.search(k + r'ILi1ELi', name) for k in KERNELS)


def test_wgmma_never_serialised(build):
    log, _ = build
    serialised = [m for m in re.findall(r'wgmma\.mma_async instructions are serialized[^\n]*\'(\S+)\'', log)
                  if any(k in m for k in KERNELS)]
    assert not serialised, 'ptxas serialises the wgmmas of %d instances, e.g. %s' % (len(serialised), serialised[0])


def test_gnn_edge_layer_takes_a_from_registers(build):
    _, funcs = build
    gnn = {n: b for n, b in funcs.items() if _is_gnn(n)}
    # 5 instruction shapes, ReLU and any-activation
    assert len(gnn) == 10, sorted(gnn)
    for name, body in gnn.items():
        hgmma = re.findall(r'HGMMA\.\S+\s+([^;]*);', body)
        assert hgmma, name
        # RS: "HGMMA.64x152x16.F32.BF16 R100, R180, gdesc[UR8], R100"; SS: "... R100, gdesc[UR16], R100"
        ss = [h for h in hgmma if not re.match(r'R\d+, R\d+, gdesc\[', h)]
        assert not ss, '%s: %d of %d HGMMAs read A from shared memory, e.g. %s' % (name, len(ss), len(hgmma), ss[0])
        sts = re.findall(r'\bSTS(?:\.\S+)?\s[^;]*;', body)
        assert not sts, '%s stores to shared memory: %s' % (name, sts[:4])
        # the __syncthreads after the mbarrier init is "BAR.SYNC.DEFER_BLOCKING 0x0"; a named barrier over one
        # warpgroup carries a thread count as a second operand
        counted = re.findall(r'\bBAR\.SYNC\S*\s+[^;,]+,[^;]*;', body)
        assert not counted, '%s syncs a warpgroup: %s' % (name, counted)

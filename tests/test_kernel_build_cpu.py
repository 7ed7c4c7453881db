"""Compile-time checks of the tensor-core kernel (no GPU needed): pg_tc.cu built with the Makefile's nvcc flags must
give every wg_gemm_kernel instance wgmmas that ptxas does not serialise (C7518) and a register budget without
spills.  A consumer warpgroup that lost its setmaxnreg registers would spill its accumulators."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'point-gnn_b200', 'csrc')


def _make_var(name):
    # the Makefile's own value of a variable (an extra makefile on stdin prints it)
    out = subprocess.run(['make', '--no-print-directory', '-s', '-C', CSRC, '-f', 'Makefile', '-f', '-', 'print-var'],
                         input='print-var:\n\t@echo $(%s)\n' % name, capture_output=True, text=True, check=True)
    return out.stdout.strip()


def test_wg_gemm_kernel_wgmma_not_serialised_and_no_spills(tmp_path):
    if shutil.which('make') is None:
        pytest.skip('make not found')
    nvcc = _make_var('NVCC')
    if not (os.path.isfile(nvcc) or shutil.which(nvcc)):
        pytest.skip('nvcc not found')
    flags = _make_var('NVCCFLAGS').split()
    assert '-v' in flags and 'arch=compute_90a,code=sm_90a' in flags
    res = subprocess.run([nvcc] + flags + ['-c', 'pg_tc.cu', '-o', str(tmp_path / 'pg_tc.o')], cwd=CSRC,
                         capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log[-4000:]

    serialised = [m for m in re.findall(r"\(C7518\)[^\n]*'(\S+)'", log) if 'wg_gemm_kernel' in m]
    assert not serialised, 'ptxas serialises the wgmmas of %d instances, e.g. %s' % (len(serialised), serialised[0])

    props = re.findall(r'Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                       r'(\d+) bytes spill loads', log)
    wg = [p for p in props if 'wg_gemm_kernel' in p[0]]
    # 3 producers x 2 epilogues, minus GNN with the store epilogue, x 5 instruction shapes
    assert len(wg) == 25, [p[0] for p in wg]
    spilled = [p for p in wg if p[2] != '0' or p[3] != '0']
    assert not spilled, 'spills in %s' % [(p[0], p[2], p[3]) for p in spilled]

"""Compile-time check of the GNN edge layer's staged P gather (no GPU needed): pg_tc.cu built with the Makefile's
nvcc flags must give every GNN instance of wg_gemm_kernel / wg_gemm_act_kernel per-thread asynchronous copies of P
into shared memory (LDGSTS) read back with LDS, and no spills."""
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


def _is_gnn(name):
    # kProd is the first template argument; PROD_GNN = 1
    return any(re.search(k + r'ILi1ELi', name) for k in KERNELS)


def test_gnn_edge_layer_gathers_p_with_cp_async_and_no_spills(tmp_path):
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
    obj = str(tmp_path / 'pg_tc.o')
    res = subprocess.run([nvcc] + flags + ['-c', 'pg_tc.cu', '-o', obj], cwd=CSRC, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log[-4000:]

    props = re.findall(r'Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                       r'(\d+) bytes spill loads', log)
    gnn_props = [p for p in props if _is_gnn(p[0])]
    assert len(gnn_props) == 10, [p[0] for p in gnn_props]
    spilled = [p for p in gnn_props if p[2] != '0' or p[3] != '0']
    assert not spilled, 'spills in %s' % [(p[0], p[2], p[3]) for p in spilled]

    sass = subprocess.run([cuobjdump, '-sass', obj], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in re.split(r'\n\s*Function : ', sass)[1:]:
        name, _, body = part.partition('\n')
        funcs[name.strip()] = body
    gnn = {n: b for n, b in funcs.items() if _is_gnn(n)}
    # 5 instruction shapes, ReLU and any-activation
    assert len(gnn) == 10, sorted(gnn)
    for name, body in gnn.items():
        assert re.search(r'\bLDGSTS\b', body), '%s: no asynchronous copy of P into shared memory' % name
        assert re.search(r'\bLDGDEPBAR\b', body), '%s: no cp.async commit group' % name
        assert re.search(r'\bLDS(?:\.\S+)?\s', body), '%s: P is never read back from shared memory' % name

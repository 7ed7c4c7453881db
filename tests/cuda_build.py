"""What nvcc makes of one CUDA source of the library, for the compile-time tests (no GPU needed).

``kernels(source)`` builds ``point-gnn_b200/csrc/build/<stem>.o`` with the Makefile (nothing to do once the library is
built, one compile on a fresh checkout) and returns one ``Kernel`` per ``__global__`` function of it: ptxas's figures
and wgmma-serialisation warnings from the log the Makefile's rule writes, and the SASS from cuobjdump.  The tests check
the object the library is linked from, built with the Makefile's own flags, once per pytest process."""
import functools
import os
import re
import shutil
import subprocess
from dataclasses import dataclass

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'point-gnn_b200', 'csrc')

# names of the template arguments of the kernel templates the tests select from
FIELDS = {'wg_gemm_kernel': ('prod', 'epi', 'ni', 'ns', 'arith', 'any_act')}


@dataclass(frozen=True)
class Kernel:
    mangled: str
    name: str            # demangled, with its template arguments and parameters
    function: str        # the name alone
    args: dict           # template arguments (a bool as 0 / 1), by FIELDS name or else by position
    registers: int
    stack: int
    spill_stores: int
    spill_loads: int
    serialised: tuple    # ptxas lines that serialise this function's wgmmas, for any reason
    sass: str


def make_var(name):
    """The Makefile's own value of a variable (an extra makefile on stdin prints it)."""
    out = subprocess.run(['make', '--no-print-directory', '-s', '-C', CSRC, '-f', 'Makefile', '-f', '-', 'print-var'],
                         input='print-var:\n\t@echo $(%s)\n' % name, capture_output=True, text=True, check=True)
    return out.stdout.strip()


@functools.lru_cache(maxsize=None)
def _cuda_bin():
    """The directory of the Makefile's nvcc, after checking the flags every compile-time test relies on."""
    if shutil.which('make') is None:
        pytest.skip('make not found')
    nvcc = make_var('NVCC')
    nvcc = nvcc if os.path.isfile(nvcc) else shutil.which(nvcc)
    if not nvcc:
        pytest.skip('nvcc not found')
    bin_dir = os.path.dirname(nvcc)
    for tool in ('cuobjdump', 'cu++filt'):
        if not os.path.isfile(os.path.join(bin_dir, tool)):
            pytest.skip('%s not found next to nvcc' % tool)
    flags = make_var('NVCCFLAGS').split()
    assert '-v' in flags and 'arch=compute_90a,code=sm_90a' in flags, flags
    return bin_dir


def _function_and_args(name):
    """'void pg::<unnamed>::f<(int)1, (bool)0>(...)' -> ('f', {FIELDS['f'][0]: 1, FIELDS['f'][1]: 0})"""
    m = re.search(r'(\w+)(?:<([^<>]*)>)?\(', name)
    vals = []
    for a in m.group(2).split(',') if m.group(2) else []:
        v = {'true': '1', 'false': '0'}.get(a.strip(), re.sub(r'^\((?:int|bool)\)', '', a.strip()))
        vals.append(int(v) if re.fullmatch(r'-?\d+', v) else v)
    return m.group(1), dict(zip(FIELDS.get(m.group(1), range(len(vals))), vals))


@functools.lru_cache(maxsize=None)
def kernels(source):
    """{mangled name: Kernel} of every __global__ function of csrc/<source>, as the Makefile builds it."""
    bin_dir = _cuda_bin()
    stem = os.path.splitext(source)[0]
    res = subprocess.run(['make', '-C', CSRC, 'build/%s.o' % stem], capture_output=True, text=True)
    assert res.returncode == 0, (res.stdout + res.stderr)[-4000:]
    with open(os.path.join(CSRC, 'build', stem + '.ptxas.log')) as f:
        log = f.read()
    sass = subprocess.run([os.path.join(bin_dir, 'cuobjdump'), '-sass', os.path.join(CSRC, 'build', stem + '.o')],
                          capture_output=True, text=True, check=True).stdout
    bodies = {}
    for part in re.split(r'\n\s*Function : ', sass)[1:]:
        name, _, body = part.partition('\n')
        bodies[name.strip()] = body
    entries = re.findall(r"Compiling entry function '(\S+)'", log)
    assert sorted(entries) == sorted(bodies), 'ptxas entries and SASS functions differ'
    demangled = subprocess.run([os.path.join(bin_dir, 'cu++filt')], input='\n'.join(entries), capture_output=True,
                               text=True, check=True).stdout.splitlines()
    serialised = [line for line in log.splitlines()
                  if re.search(r'\(C75\d\d\)|wgmma\.mma_async instructions are serialized', line)]
    out = {}
    for mangled, name in zip(entries, demangled):
        props = re.search(r'Function properties for %s\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                          r'(\d+) bytes spill loads' % re.escape(mangled), log)
        regs = re.search(r"Compiling entry function '%s'.*?Used (\d+) registers" % re.escape(mangled), log, re.S)
        assert props and regs, mangled
        out[mangled] = Kernel(mangled, name, *_function_and_args(name), int(regs.group(1)), int(props.group(1)),
                              int(props.group(2)), int(props.group(3)),
                              tuple(line for line in serialised if "'%s'" % mangled in line), bodies[mangled])
    return out

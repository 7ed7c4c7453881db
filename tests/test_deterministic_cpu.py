"""PG_FLAG_DETERMINISTIC without a GPU: the header and the Python constant agree and the bit is free; the library
rejects it where it has no meaning and with an unknown aggregation code, before it touches the device; _lib sets it
exactly while torch.use_deterministic_algorithms(True) is in force; and the ordered instances of the tensor-core edge
kernel (wg_segsum_ordered_kernel) are all there, free of spills, serialised wgmmas and floating-point atomics."""
import concurrent.futures
import ctypes
import os
import re

import pytest
import torch

import cuda_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from pointgnn_b200 import _lib
    return _lib


def test_header_macro_and_python_constant_agree():
    lib = _lib()
    with open(os.path.join(ROOT, 'include', 'pointgnn_b200.h')) as f:
        text = f.read()
    m = re.search(r'#define PG_FLAG_DETERMINISTIC (0x[0-9a-f]+)\b', text)
    assert m and lib.PG_FLAG_DETERMINISTIC == int(m.group(1), 16)
    bit = lib.PG_FLAG_DETERMINISTIC
    assert bin(bit).count('1') == 1
    for taken in (lib.PG_PRECISION_MASK, lib.PG_FLAG_TRUSTED_INDICES, lib.PG_FLAG_ACTIVATION, lib.PG_ACT_MASK,
                  lib.PG_AGG_MASK, lib.PG_FLAG_SEPARATED):
        assert taken & bit == 0
    assert lib.PG_ORDERED_SCATTER_TILE == 64


class _Lib(object):
    """The library itself: argument checks return before any CUDA call, so no GPU is needed.  Each call runs on a
    thread of its own and returns (status, that thread's pg_last_error), so the error text it sets stays there."""

    def __init__(self):
        self._lib = _lib().load()

    def __getattr__(self, name):
        fn = getattr(self._lib, name)

        def call(*args):
            def run():
                return fn(*args), self._lib.pg_last_error().decode()
            with concurrent.futures.ThreadPoolExecutor(1) as pool:
                return pool.submit(run).result()
        return call


@pytest.fixture
def clib():
    return _Lib()


def _edge_call(clib, flags):
    null = (ctypes.c_void_p * 1)()
    dims = (ctypes.c_int32 * 3)(6, 8, 8)
    return clib.pg_edge_mlp_max(1, None, 3, None, None, None, None, None, 0, 1, 0, null, null, dims, 2, None, flags,
                                None)


def test_bit_rejected_with_an_unknown_aggregation(clib):
    lib = _lib()
    det = lib.PG_FLAG_DETERMINISTIC
    rc, error = _edge_call(clib, 1 | (3 << lib.PG_AGG_SHIFT) | det)
    assert rc == lib.PG_ERR_INVALID_ARGUMENT and 'unknown aggregation' in error
    # with a known aggregation the bit passes the flag checks (the call then stops at its null weights)
    rc, error = _edge_call(clib, 1 | (1 << lib.PG_AGG_SHIFT) | det)
    assert rc == lib.PG_ERR_INVALID_ARGUMENT and 'null weight' in error


def test_bit_rejected_where_it_means_nothing(clib):
    lib = _lib()
    det = lib.PG_FLAG_DETERMINISTIC
    null = (ctypes.c_void_p * 1)()
    dims = (ctypes.c_int32 * 2)(8, 8)
    handle = ctypes.c_void_p()
    rc, error = clib.pg_layer_create(lib.PG_LAYER_EDGE_GNN, null, null, dims, 1, 1 | det, None, ctypes.byref(handle))
    assert rc == lib.PG_ERR_INVALID_ARGUMENT and 'PG_FLAG_DETERMINISTIC' in error and not handle.value
    fake = ctypes.c_void_p(256)    # never dereferenced: the precision word is checked first
    rc, error = clib.pg_fully_connected(fake, 1, 8, fake, fake, 8, 0, None, fake, 1 | det, None)
    assert rc == lib.PG_ERR_INVALID_ARGUMENT and 'precision' in error
    # pg_scatter_sum_flags / _mean_flags take the bit and nothing else; pg_scatter_sum / _mean keep their signatures
    for name in ('pg_scatter_sum', 'pg_scatter_mean'):
        assert [n for _, n in lib.PROTOTYPES[name][1]][-2:] == ['out', 'stream']
    for name in ('pg_scatter_sum_flags', 'pg_scatter_mean_flags'):
        for flags in (0x1, lib.PG_FLAG_TRUSTED_INDICES, det | (1 << lib.PG_AGG_SHIFT)):
            rc, error = getattr(clib, name)(None, None, 0, 4, 0, None, flags, None)
            assert rc == lib.PG_ERR_INVALID_ARGUMENT and 'unknown flags' in error
        assert getattr(clib, name)(None, None, 0, 4, 0, None, det, None) == (lib.PG_OK, '')


@pytest.fixture
def calls(monkeypatch):
    """The flag words _lib passes, by function, with the library replaced by a recorder."""
    lib = _lib()
    seen = []

    def record(function, error=None, **args):
        seen.append((function, args.get('flags', args.get('precision'))))
        return 0

    monkeypatch.setattr(lib, '_call', record)
    was, was_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield seen
    torch.use_deterministic_algorithms(was, warn_only=was_warn)


def _every_call(lib):
    feat, idx = torch.zeros(6, 2), torch.zeros(6, dtype=torch.int32)
    lib.scatter_sum(feat, idx, 3)
    lib.scatter_sum(feat, idx, 3, mean=True)
    w = [torch.zeros(5, 8), torch.zeros(8, 8)]
    for aggregation in ('max', 'sum', 'mean'):
        lib.edge_mlp_max(1, feat, None, None, None, idx, idx, 3, w, w, precision=1, aggregation=aggregation)
        layer = object.__new__(lib.PreparedLayer)
        layer._handle, layer.dims = None, [5, 8, 8]
        layer.edge_mlp_max(feat, None, None, None, idx, idx, 3, aggregation=aggregation)


@pytest.mark.parametrize('mode', ['off', 'on', 'warn_only'])
def test_lib_sets_the_bit_exactly_under_the_switch(mode, calls):
    lib = _lib()
    torch.use_deterministic_algorithms(mode != 'off', warn_only=mode == 'warn_only')
    _every_call(lib)
    assert [f for f, _ in calls] == ['pg_scatter_sum_flags', 'pg_scatter_mean_flags'] + \
        ['pg_edge_mlp_max', 'pg_layer_edge_mlp_max'] * 3
    want = lib.PG_FLAG_DETERMINISTIC if mode != 'off' else 0
    assert all(flags & lib.PG_FLAG_DETERMINISTIC == want for _, flags in calls), calls


# ---- compile-time checks of the ordered instances ---------------------------------------------------------------------
PROD_ROWS, PROD_GNN, PROD_POOL = 0, 1, 2
SHAPES = ((64, 1), (128, 1), (96, 2), (128, 2), (152, 2))


def _ordered():
    return [k for k in cuda_build.kernels('pg_tc.cu').values() if k.function == 'wg_segsum_ordered_kernel']


def test_ordered_instance_census():
    want = sorted((prod, ni, ns, arith, act) for arith in (0, 1) for ni, ns in SHAPES
                  for prod, act in ((PROD_ROWS, 0), (PROD_POOL, 0), (PROD_GNN, 0), (PROD_GNN, 1)))
    got = sorted(tuple(k.args[i] for i in range(5)) for k in _ordered())
    assert len(want) == 40 and got == want, got


def test_ordered_instances_compile_clean():
    """No serialised wgmmas, no spills, and no floating-point atomics: every partial sum is stored."""
    ks = _ordered()
    assert len(ks) == 40
    serialised = [line for k in ks for line in k.serialised]
    assert not serialised, serialised[:1]
    spilled = [(k.name, k.spill_stores, k.spill_loads) for k in ks if k.spill_stores or k.spill_loads]
    assert not spilled, spilled
    for k in ks:
        assert not re.search(r'\b(?:RED|ATOM)G?\.E\.ADD\.F32', k.sass), k.name

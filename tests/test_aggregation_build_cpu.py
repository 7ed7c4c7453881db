"""Compile-time checks of the segment-sum instances of the tensor-core edge kernel (no GPU needed):
wg_segsum_kernel<prod, ni, ns, arith, any_act>, wg_gemm_kernel's bodies with the EPI_SEGSUM epilogue.  The same checks
tests/test_tc_build_cpu.py makes of wg_gemm_kernel: no serialised wgmmas, no spills (the sum applies bias and
activation to every accumulator before it reduces), A in registers and P gathered with cp.async in the GNN edge layer,
and the HGMMA input type of each arithmetic."""
import re

import cuda_build

PROD_ROWS, PROD_GNN, PROD_POOL = 0, 1, 2
ARITH_BF16X3, ARITH_F16 = 0, 1
SHAPES = ((64, 1), (128, 1), (96, 2), (128, 2), (152, 2))   # ni, ns
FIELDS = ('prod', 'ni', 'ns', 'arith', 'any_act')


def _instances(**fields):
    out = []
    for k in cuda_build.kernels('pg_tc.cu').values():
        if k.function == 'wg_segsum_kernel':
            args = dict(zip(FIELDS, k.args.values()))
            if all(args[f] == v for f, v in fields.items()):
                out.append((args, k))
    return out


def test_instance_census():
    # per arithmetic and instruction shape: the ped pooling split's row launch, the pooling chain, and the GNN edge
    # layer with ReLU and with any activation
    want = sorted((prod, ni, ns, arith, act) for arith in (ARITH_BF16X3, ARITH_F16) for ni, ns in SHAPES
                  for prod, act in ((PROD_ROWS, 0), (PROD_POOL, 0), (PROD_GNN, 0), (PROD_GNN, 1)))
    got = sorted(tuple(a.values()) for a, _ in _instances())
    assert len(want) == 40 and got == want, got


def test_wgmma_not_serialised_and_no_spills():
    ks = [k for _, k in _instances()]
    assert len(ks) == 40
    serialised = [line for k in ks for line in k.serialised]
    assert not serialised, 'ptxas serialises the wgmmas of %d instances, e.g. %s' % (len(serialised), serialised[0])
    spilled = [(k.name, k.spill_stores, k.spill_loads) for k in ks if k.spill_stores or k.spill_loads]
    assert not spilled, 'spills in %s' % spilled


def test_gnn_edge_layer_takes_a_from_registers_and_gathers_p_with_cp_async():
    gnn = [k for _, k in _instances(prod=PROD_GNN)]
    assert len(gnn) == 20
    for k in gnn:
        hgmma = re.findall(r'HGMMA\.\S+\s+([^;]*);', k.sass)
        assert hgmma and all(re.match(r'R\d+, R\d+, gdesc\[', h) for h in hgmma), k.name
        assert not re.findall(r'\bSTS(?:\.\S+)?\s[^;]*;', k.sass), k.name
        assert re.search(r'\bLDGSTS\b', k.sass) and re.search(r'\bLDGDEPBAR\b', k.sass), k.name


def test_hgmma_input_type_follows_the_arithmetic():
    def kinds(sass):
        return [t or 'F16' for t in re.findall(r'HGMMA\.\d+x\d+x16\.F32(?:\.(\w+))?\s', sass)]
    count = {}
    for arith, want in ((ARITH_BF16X3, 'BF16'), (ARITH_F16, 'F16')):
        ks = [k for _, k in _instances(arith=arith)]
        assert len(ks) == 20
        for k in ks:
            assert set(kinds(k.sass)) == {want}, (k.name, sorted(set(kinds(k.sass))))
        count[arith] = sum(len(kinds(k.sass)) for k in ks)
    assert count[ARITH_BF16X3] == 3 * count[ARITH_F16], count


def test_sum_atomics_only_in_the_sum_instances():
    """The sum flushes with fp32 atomic adds (REDG.E.ADD.F32); the max's instances keep their integer atomics only."""
    for _, k in _instances():
        assert re.search(r'\bREDG\.E\.ADD\.F32', k.sass), k.name
    for k in cuda_build.kernels('pg_tc.cu').values():
        if k.function == 'wg_gemm_kernel':
            assert not re.search(r'\bREDG\.E\.ADD\.F32', k.sass), k.name

"""Compile-time checks of the tensor-core kernel (no GPU needed), on the pg_tc.cu object the Makefile builds.

Every instance of wg_gemm_kernel<prod, epi, ni, ns, arith, any_act> is selected by its template arguments, and each
check runs on every instance it concerns: ptxas must not serialise any instance's wgmmas, for any reason, nor spill
(a consumer warpgroup that lost its setmaxnreg registers would spill its accumulators); the GNN edge layer builds A
in registers and gathers its rows of P into shared memory with cp.async; and every HGMMA takes the input type of
its instance's arithmetic."""
import re

import cuda_build

# pg_tc.cu's enums
PROD_ROWS, PROD_GNN, PROD_POOL = 0, 1, 2
EPI_STORE, EPI_SEGMAX = 0, 1
ARITH_BF16X3, ARITH_F16 = 0, 1
SHAPES = ((64, 1), (128, 1), (96, 2), (128, 2), (152, 2))   # ni, ns


def _instances(**fields):
    """The wg_gemm_kernel instances whose template arguments equal fields."""
    return [k for k in cuda_build.kernels('pg_tc.cu').values()
            if k.function == 'wg_gemm_kernel' and all(k.args[f] == v for f, v in fields.items())]


def test_instance_census():
    # per arithmetic: ROWS and POOL with either epilogue, and the GNN edge layer with the segment max, ReLU and any
    # activation, each at every instruction shape
    want = []
    for arith in (ARITH_BF16X3, ARITH_F16):
        for ni, ns in SHAPES:
            want += [(prod, epi, ni, ns, arith, 0) for prod in (PROD_ROWS, PROD_POOL) for epi in (EPI_STORE, EPI_SEGMAX)]
            want += [(PROD_GNN, EPI_SEGMAX, ni, ns, arith, any_act) for any_act in (0, 1)]
    got = sorted(tuple(k.args.values()) for k in _instances())
    assert len(want) == 60 and got == sorted(want), got


def test_wgmma_not_serialised_and_no_spills():
    wg = _instances()
    assert len(wg) == 60
    serialised = [line for k in wg for line in k.serialised]
    assert not serialised, 'ptxas serialises the wgmmas of %d instances, e.g. %s' % (len(serialised), serialised[0])
    spilled = [(k.name, k.spill_stores, k.spill_loads) for k in wg if k.spill_stores or k.spill_loads]
    assert not spilled, 'spills in %s' % spilled


def test_gnn_edge_layer_takes_a_from_registers():
    gnn = _instances(prod=PROD_GNN)
    assert len(gnn) == 20
    for k in gnn:
        hgmma = re.findall(r'HGMMA\.\S+\s+([^;]*);', k.sass)
        assert hgmma, k.name
        # RS: "HGMMA.64x152x16.F32.BF16 R100, R180, gdesc[UR8], R100"; SS: "... R100, gdesc[UR16], R100"
        ss = [h for h in hgmma if not re.match(r'R\d+, R\d+, gdesc\[', h)]
        assert not ss, '%s: %d of %d HGMMAs read A from shared memory, e.g. %s' % (k.name, len(ss), len(hgmma), ss[0])
        sts = re.findall(r'\bSTS(?:\.\S+)?\s[^;]*;', k.sass)
        assert not sts, '%s stores to shared memory: %s' % (k.name, sts[:4])
        # the __syncthreads after the mbarrier init is "BAR.SYNC.DEFER_BLOCKING 0x0"; a named barrier over one
        # warpgroup carries a thread count as a second operand
        counted = re.findall(r'\bBAR\.SYNC\S*\s+[^;,]+,[^;]*;', k.sass)
        assert not counted, '%s syncs a warpgroup: %s' % (k.name, counted)


def test_gnn_edge_layer_gathers_p_with_cp_async():
    gnn = _instances(prod=PROD_GNN)
    assert len(gnn) == 20
    for k in gnn:
        assert re.search(r'\bLDGSTS\b', k.sass), '%s: no asynchronous copy of P into shared memory' % k.name
        assert re.search(r'\bLDGDEPBAR\b', k.sass), '%s: no cp.async commit group' % k.name
        assert re.search(r'\bLDS(?:\.\S+)?\s', k.sass), '%s: P is never read back from shared memory' % k.name


def test_hgmma_input_type_follows_the_arithmetic():
    # the SASS of an HGMMA names its input type after the accumulator's, except FP16, the default:
    # "HGMMA.64x152x16.F32 ..." is FP16, "HGMMA.64x152x16.F32.BF16 ..." BF16
    def kinds(sass):
        return [t or 'F16' for t in re.findall(r'HGMMA\.\d+x\d+x16\.F32(?:\.(\w+))?\s', sass)]
    count = {}
    for arith, want in ((ARITH_BF16X3, 'BF16'), (ARITH_F16, 'F16')):
        wg = _instances(arith=arith)
        assert len(wg) == 30
        for k in wg:
            assert set(kinds(k.sass)) == {want}, (k.name, sorted(set(kinds(k.sass))))
        count[arith] = sum(len(kinds(k.sass)) for k in wg)
    # BF16x3 issues three HGMMAs for every FP16 one
    assert count[ARITH_BF16X3] == 3 * count[ARITH_F16], count

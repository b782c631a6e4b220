"""The shared-memory node kernel (k_node_batch, jslp_node_kernel.cuh) and the single-CTA branch-and-cut primitives at the
edges of their geometry, bit for bit against the oracle.

The node kernel restates every simplex rule at warp scope: phase-2 pricing dealt over 32 lanes in partial-pricing
batches, the phase-1 leaving row scanned by one warp, the ratio test and the phase-1 column scan reduced from one
partial per warp, the division pass split between the pivot row and the pivot column, the row update in column
blocks.  Every LP here runs on engine 4 (the node kernel) at widths and heights on both sides of those splits, with
the mixed, tie and threshold value families of test_gpu_shape_edges.py, and pivots in both phases.

k_mip_scan (isIntegral / getMostFractionalVar), k_add_cuts (addCutConstraints) and k_mir_cuts (the MIR cuts) are one
256-thread CTA each: they run here on uploaded tableaux taller and wider than one pass of that CTA, with exact fraction
ties, values on the precision thresholds and signed zeros."""
import types

import numpy as np
import pytest

from test_gpu_lp_parity import assert_lp_parity, gpu_lp, oracle_lp, same_bits
from test_gpu_shape_edges import device, resident_rows, solved

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------ the node kernel's geometry, restated
NODE_THREADS = 256      # jslp_node_kernel.cuh:106 (NODE_THREADS): 8 warps, one partial each in S2 / S3 (:384, :406)
NODE_WARPS = NODE_THREADS // 32
D_SPLIT = NODE_THREADS // 2   # jslp_node_kernel.cuh:453: threads below NT / 2 normalise the pivot row, the rest the column
U_BLOCK = 128           # jslp_node_kernel.cuh:473: the row update walks the columns in blocks of 4 x 32
PRICE_BATCH = 50        # jslp_api.cu:248: smallest partial-pricing batch; on while W - 1 > 2 x batch (:250)
NODE_LOG_HEAD = 64      # jslp_node_kernel.cuh:34: pivot-log entries a CTA reports inline

MIXED = (4, 20)          # mixed_arrays(n_lower=4, profitable=20): few phase-2 pivots at any width
# (family, H, W, seed, extra); H = "resident": the tallest tableau the node kernel takes at width W.  Seeds: the first
# from 9000 on which the oracle pivots in both phases (the reference's phase-1 rule runs very long on some instances)
K2_CASES = [
    ("mixed", 32, 32, 9000, MIXED), ("mixed", 33, 33, 9000, MIXED),            # one lane pass; phase-1 warp scan
    ("mixed", 33, 51, 9000, MIXED), ("mixed", 32, 52, 9000, MIXED),            # 50 / 51 priced columns
    ("mixed", 128, 33, 9000, MIXED), ("mixed", 129, 32, 9001, MIXED),          # D pass: 128 / 129 rows
    ("mixed", 128, 129, 9001, MIXED), ("mixed", 129, 128, 9000, MIXED),        # U block: 128 / 129 columns
    ("mixed", 256, 52, 9001, MIXED), ("mixed", 257, 51, 9000, MIXED),          # a second ratio-test pass per thread
    ("mixed", 33, 257, 9000, MIXED), ("mixed", "resident", 257, 9000, MIXED),  # three U blocks, two column-scan passes
    ("mixed", "resident", 33, 9001, MIXED),
    # ties: tableau rows 2..9 copied 32 rows on (another warp's partial) and 256 on (the same thread, a later pass);
    # the top-cost column copied 50 columns on (the same pricing batch below 101 columns, another lane), 32 on (the
    # same lane, next pass) and 128 on (the next U block; the next pricing batch at 257 columns)
    ("ties", 289, 60, 9001, (1, NODE_THREADS, 20, (32, 256), (PRICE_BATCH, 32))),
    ("ties", 100, 257, 9000, (1, NODE_THREADS, 20, (32, 64), (PRICE_BATCH, 32, U_BLOCK))),
    ("thresholds", 129, 60, 9000, ()), ("thresholds", 257, 33, 9000, ()), ("thresholds", 100, 257, 9000, ()),
]


def _k2_id(case):
    fam, H, W = case[:3]
    return f"{fam}-{H}x{W}"


@pytest.mark.parametrize("case", K2_CASES, ids=[_k2_id(c) for c in K2_CASES])
def test_node_kernel_at_its_edges(case):
    family, H, W, seed, extra = case
    dev = device()
    if H == "resident":
        H = resident_rows(dev, W)
    assert H <= resident_rows(dev, W), (H, W)
    it, o = solved(family, H - 1, W - 1, seed, extra)
    g = gpu_lp(it, 4)
    g.simplex()
    st = g.lastStatus
    what = f"K2 {family} {H}x{W}"
    print(f"{what}: engine {st.engine} pivots {st.phase1_pivots}+{st.phase2_pivots}")
    assert st.engine == 4, (what, st.engine)
    assert_lp_parity(g, o, what)
    assert st.phase1_pivots > 0 and st.phase2_pivots > 0, (what, st.phase1_pivots, st.phase2_pivots)
    if family == "ties" and W == 60:
        assert st.phase1_pivots + st.phase2_pivots > NODE_LOG_HEAD   # the log is read back past the inline head
    g.close()


# ------------------------------------------------------------------ a tie LP through the other node-kernel modes
TIE_SMALL = (1, NODE_THREADS, 20, (32, 128), (PRICE_BATCH, 32))   # 161 x 100: H x W <= 16 384, the automatic engine's K2


def test_scenarios_on_a_tied_lp_match_the_sequential_path():
    """scenarios() on the tie family: every scenario of the shared-memory batch equals the sequential device path and
    the oracle (test_gpu_scenarios.assert_batch)."""
    from test_gpu_scenarios import _picks, _tableau, assert_batch
    it, _ = solved("ties", 160, 99, 9000, TIE_SMALL)
    g = _tableau(it)
    assert g.lastStatus.engine == 4 and g.feasible and g.bounded
    sc = _picks(g, it, np.random.default_rng(5), 10) + [[]]
    assert_batch(it, g, sc, what="ties 161x100")
    g.close()


def test_deletion_filter_sets_on_a_tied_lp_match_the_oracle():
    """The sets an IIS deletion filter tests (the whole row set, then one row dropped at a time) and random subsets of
    the tie family, as one shared-memory feasibility batch: verdict and phase-1 pivot count of the oracle's filter."""
    from test_gpu_iis import _check_batch, _random_sets
    it, _ = solved("ties", 160, 99, 9000, TIE_SMALL)
    H = it.matrix.shape[0]
    sets = [list(range(1, H))] + [[r for r in range(1, H) if r != s] for s in range(1, 40)]
    sets += _random_sets(H, 16, np.random.default_rng(6), p=0.9)
    _check_batch(it, 1e-8, sets, "ties 161x100")


# ------------------------------------------------------------------ k_mip_scan on uploaded tableaux
def crafted(M, vrow, vcol, ints):
    """An upload source (the fields gpu_lp / oracle_lp read) for a hand-made tableau."""
    H, W = M.shape
    return types.SimpleNamespace(matrix=np.ascontiguousarray(M, dtype=np.float64), varIndexByRow=np.asarray(vrow, np.int32),
                                 varIndexByCol=np.asarray(vcol, np.int32), unrestricted=np.zeros(H + W - 2, np.uint8),
                                 integerIndices=np.asarray(ints, np.int32), optionalCosts=np.zeros((0, W)))


ULP_HALF = [np.nextafter(0.5, 0.0), np.nextafter(0.5, 1.0), np.nextafter(2.5, 0.0), np.nextafter(-1.5, 0.0)]
PREC = 1e-8
MIP_VALUES = {
    # exact k + 1/2 everywhere: the branching variable is decided by position alone
    "ties": lambda rng, n: rng.integers(-3, 4, n) + 0.5,
    # k + 1/2 next to 1/2 +- 1 ulp, values >= 2^52 (2^52 - 1/2 is the last half), negative halves (Math.round goes
    # toward +inf), signed zeros, subnormals and the precision threshold
    "edges": lambda rng, n: rng.choice(np.array(ULP_HALF + [2.0 ** 52 - 0.5, 2.0 ** 52 + 1.0, 2.0 ** 53, -2.5, -0.5, 0.5,
                                                            3.5, 0.0, -0.0, 5e-324, -1e-310, PREC, 7.0, -3.0, 1e300]), n),
    # integral values and one value on the precision: at / just under / just over it (isIntegral changes at the last)
    "prec_at": lambda rng, n: rng.integers(-3, 4, n).astype(np.float64),
    "prec_under": lambda rng, n: rng.integers(-3, 4, n).astype(np.float64),
    "prec_over": lambda rng, n: rng.integers(-3, 4, n).astype(np.float64),
}
PREC_VALUE = {"prec_at": PREC, "prec_under": np.nextafter(PREC, 0.0), "prec_over": np.nextafter(PREC, 1.0)}


def mip_scan_tableau(H, kind, seed):
    """H x 6 tableau whose basic variables in about 2 of 3 rows are integer, plus 3 non-basic integer variables (their
    values are not read), integerIndices in an order unrelated to the rows with one entry repeated."""
    rng = np.random.default_rng(seed)
    W = 6
    n_index = H + W - 2
    labels = rng.permutation(n_index).astype(np.int32)
    vrow = np.concatenate([[-1], labels[:H - 1]])
    vcol = np.concatenate([[-1], labels[H - 1:]])
    M = rng.integers(-9, 10, size=(H, W)).astype(np.float64)
    rows = np.array([r for r in range(1, H) if r % 3 != 1 or r == H - 1 or r > 256], dtype=int)
    M[rows, 0] = MIP_VALUES[kind](rng, len(rows))
    if kind in PREC_VALUE:
        M[rows[-1], 0] = PREC_VALUE[kind]              # the last integer row: past 256 where H allows
    ints = list(vrow[rows]) + list(vcol[1:4])
    ints = [int(v) for v in rng.permutation(np.array(ints, dtype=np.int32))]
    ints.insert(len(ints) // 2, ints[-1])            # a duplicate entry: its first position counts
    return crafted(M, vrow, vcol, ints)


MIP_SCAN_CASES = [(H, kind) for H in (2, 33, 256, 257, 258, 1025) for kind in ("ties", "edges")]
MIP_SCAN_CASES += [(258, k) for k in PREC_VALUE] + [(1025, k) for k in PREC_VALUE]


@pytest.mark.parametrize("H,kind", MIP_SCAN_CASES, ids=[f"H{h}-{k}" for h, k in MIP_SCAN_CASES])
def test_mip_scan_on_uploaded_tableaux(H, kind):
    """isIntegral and getMostFractionalVar (mip-utils.ts:43-61,100-126) over 1 .. 4 passes of the 256-thread scan:
    the flag, the variable index and the bits of its value."""
    it = mip_scan_tableau(H, kind, 100 + H)
    o = oracle_lp(it)
    g = gpu_lp(it, 2)
    iv, val = o.most_fractional()
    mf = g.getMostFractionalVar()
    got = -1 if mf["index"] is None else mf["index"]
    print(f"H{H} {kind}: integral {o.is_integral()} most fractional {iv} = {val!r}")
    assert g.isIntegral() == o.is_integral(), (H, kind)
    assert got == iv and same_bits(mf["value"], val), (H, kind, got, mf["value"], iv, val)
    if kind in PREC_VALUE:
        assert o.is_integral() == (kind != "prec_over")
    g.close()


# ------------------------------------------------------------------ k_add_cuts and k_mir_cuts on uploaded tableaux
def solved_source(H, W, seed, ints=()):
    """The oracle's optimal tableau of a mixed LP as an upload source (a fresh copy: the cached oracle stays as is)."""
    _, o = solved("mixed", H - 1, W - 1, seed, MIXED)
    vr, vc = o.maps()
    return crafted(o.matrix().copy(), vr.copy(), vc.copy(), list(ints))


def upload(it, row_capacity=None, engine=2):
    from jslpsolver_b200 import _lib
    from jslpsolver_b200.tableau import GpuTableau
    g = GpuTableau(1e-8)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, it.integerIndices, it.optionalCosts,
             row_capacity=row_capacity)
    g.set_option(_lib.OPT_ENGINE, engine)
    g.set_option(_lib.OPT_PIVOT_LOG_CAP, 1 << 16)
    return g


def assert_same_tableau(g, o, what):
    assert g.height == o.state().height, (what, g.height, o.state().height)
    assert np.array_equal(g.varIndexByRow, o.maps()[0]) and np.array_equal(g.varIndexByCol, o.maps()[1]), what
    assert same_bits(g.matrix2d(), o.matrix()), f"{what}: tableau bits differ"


@pytest.mark.parametrize("W", [255, 256, 257, 600])
def test_add_cuts_past_one_cta_pass(W):
    """addCutConstraints (cutting-strategies.ts:36-71) on a 300-row optimal tableau: cuts of both types on variables
    basic in rows past 256 and non-basic in the last columns (past 256 at W = 600), more cuts than the spare row
    capacity (the rows grow), then a re-solve with parity."""
    H = 300
    it = solved_source(H, W, 9001 if W == 257 else 9000)   # the first seed from 9000 whose LP solves quickly
    vr, vc = it.varIndexByRow, it.varIndexByCol
    cuts = []
    for r in (257, 270, H - 1):   # a loose pair, then a bound that cuts the optimum off
        v = float(it.matrix[r, 0])
        cuts += [("min", int(vr[r]), np.floor(v)), ("max", int(vr[r]), np.floor(v) + 1.0)]
    cuts.append(("max", int(vr[H - 1]), np.floor(float(it.matrix[H - 1, 0])) - 1.0))
    for c in (W - 1, W - 2, 257 if W > 258 else 200):
        cuts += [("min", int(vc[c]), 1.0), ("max", int(vc[c]), 2.0)]
    o = oracle_lp(it)
    g = upload(it, row_capacity=H + 4)
    o.add_cuts(cuts)
    g.addCutConstraints(cuts)
    assert_same_tableau(g, o, f"cuts W{W}")
    o.simplex()
    g.simplex()
    assert_lp_parity(g, o, f"after cuts W{W}")
    g.close()


# right-hand sides of the rows past 256 that the MIR tests set: (value, eligible)
_ONE_M = 1.0 - PREC
MIR_RHS = [(PREC, True), (np.nextafter(PREC, 1.0), True), (np.nextafter(PREC, 0.0), False),
           (_ONE_M, True), (np.nextafter(_ONE_M, 0.0), True), (np.nextafter(_ONE_M, 1.0), False),
           (2.5, True), (3.0, False), (7.25, True), (0.75, True), (-1.5, True), (11.0, False), (4.125, True),
           (1.0 + 2.0 ** -30, False), (1.0 + 2.0 ** -20, True), (6.5, True), (9.875, True), (5.5, True), (2.0 ** 40 + 0.5, True)]


def mir_tableau(seed=9000):
    """A 300 x 300 optimal tableau of a mixed LP with the rows from 260 on holding integer basic variables whose
    right-hand sides are MIR_RHS (more than 10 eligible; fractions exactly prec and 1 - prec and one ulp either side),
    integer non-basic variables in columns past 256 and before, and entries -0, +0 and negative in those rows."""
    H = W = 300
    it = solved_source(H, W, seed)
    rows = list(range(260, 260 + len(MIR_RHS)))
    M = it.matrix
    for r, (v, _) in zip(rows, MIR_RHS):
        M[r, 0] = v
        M[r, 258:262] = [-0.0, 0.0, -2.75, -0.0]         # integer columns past 256
        M[r, 3:7] = [-0.0, 0.0, -1.25, -3.0]             # columns 3, 4: integer; 5, 6: not
    ints = [int(it.varIndexByRow[r]) for r in rows] + [int(it.varIndexByCol[c]) for c in (258, 259, 260, 261, 3, 4)]
    it.integerIndices = np.asarray(np.random.default_rng(seed).permutation(ints), np.int32)
    return it, rows


def test_apply_mir_cuts_takes_the_first_ten_eligible_rows_past_256():
    """applyMIRCuts (cutting-strategies.ts:198-212): every eligible row lies in the scan's second 256-row pass and
    there are more than 10; the cut rows are those of the first 10 in row order.  Then a re-solve with parity."""
    it, rows = mir_tableau()
    eligible = [r for r, (_, ok) in zip(rows, MIR_RHS) if ok]
    assert len(eligible) > 10
    o = oracle_lp(it)
    g = upload(it)
    assert o.apply_mir_cuts() == 10
    g.applyMIRCuts()
    assert_same_tableau(g, o, "applyMIRCuts")
    o.simplex()
    g.simplex()
    assert_lp_parity(g, o, "after applyMIRCuts")
    g.close()


def test_mir_cut_rows_past_256():
    """addLowerBoundMIRCut / addUpperBoundMIRCut on every crafted row past 256 (eligible or not, fractions on and next
    to prec and 1 - prec, -0 / +0 / negative coefficients through Math.min(0, .) and Math.max(0, .)), then a re-solve
    with parity."""
    it, rows = mir_tableau()
    o = oracle_lp(it)
    g = upload(it)
    for r, (_, ok) in zip(rows, MIR_RHS):
        assert g.addLowerBoundMIRCut(r) == o.add_mir_cut(r) == ok, r
        assert g.addUpperBoundMIRCut(r) == o.add_mir_cut(r, upper=True) == ok, r
    assert_same_tableau(g, o, "MIR cut rows")
    o.simplex()
    g.simplex()
    assert_lp_parity(g, o, "after MIR cut rows")
    g.close()


# ------------------------------------------------------------------ the node kernel's shared-memory limit
def test_node_kernel_limit_is_shared_by_tabs_of_different_heights():
    """The dynamic shared-memory limit of k_node_batch belongs to the kernel on the device, not to a tab: a resident LP
    (engine 4) on a short tab between two branch and cuts of a tall tab on the same context leaves the second branch and
    cut equal to the first, node log and final column bit for bit."""
    import ctypes as C
    from jslpsolver_b200 import _lib, problems
    from jslpsolver_b200.model import Model
    from jslpsolver_b200.tableau import GpuTableau
    model = Model().loadJson(dict(problems.knapsack_mip_model(40, 100, seed=21), options={"presolve": False}))
    it = model.initial_tableau()
    assert it.matrix.shape == (141, 41) and not np.any(it.unrestricted)  # node CTAs above 48 KB of shared memory
    tall = GpuTableau(model.precision)
    tall.setModel(model)
    ints = np.ascontiguousarray(it.integerIndices, dtype=np.int32)

    def branch_and_cut():
        # the same jslp_tab back at the initial tableau: restore() brings back the root's height, the upload its content
        tall.restore()
        M, vrow, vcol = (np.ascontiguousarray(a, dtype=d) for a, d in
                         ((it.matrix, np.float64), (it.varIndexByRow, np.int32), (it.varIndexByCol, np.int32)))
        _lib.check(tall.context.lib.jslp_tab_upload(tall._h(), M.ctypes.data, vrow.ctypes.data, vcol.ctypes.data, None,
                                                    M.shape[0] + M.shape[1] - 2, ints.ctypes.data, len(ints), 0, None))
        tall.branchAndCut()
        st = tall.lastBnbStatus
        assert st.node_kernel_ms > 0  # rounds ran in the node kernel
        counters = tuple(getattr(st, f) for f in ("feasible", "bounded", "is_integral", "iterations", "n_best_cuts",
                                                   "rounds", "nodes_evaluated", "pivots", "kernel_launches"))
        return counters, np.float64(st.evaluation).tobytes(), tall.node_log().tobytes(), tall.rhs_column().tobytes()

    first = branch_and_cut()
    short = GpuTableau(1e-8, context=tall.context)
    lp = problems.dense_packing_lp_tableau(8, 6, seed=5)
    short.upload(lp.matrix, lp.varIndexByRow, lp.varIndexByCol)
    short.set_option(_lib.OPT_ENGINE, _lib.ENGINE_RESIDENT)
    short.simplex()
    assert short.lastStatus.engine == _lib.ENGINE_RESIDENT
    assert branch_and_cut() == first
    short.close()
    tall.close()

"""GPU checks of the warm start (DESIGN.md section 2f): jslp_crash's records, the tableau it leaves (every fp64 entry),
the row and column labels, and the simplex() that follows (its pivot log, flags and evaluation) equal the oracle
restatement bit for bit, with engines 0, 1, 2 and 4 -- on every continuous fixture (round trip), on seeded edited LPs,
on a tableau beyond shared memory, on config 3 from its stored optimal basis, and at the geometry edges of
k_crash_select; Solve(basis=...) returns the oracle's result dict."""
import numpy as np
import pytest

from conftest import load_bundle
from helpers import strip_timeouts

pytestmark = pytest.mark.gpu
BUNDLE = load_bundle()
ENGINES = [0, 1, 2, 4]
P = 1e-8


def _soft(jm):
    return any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())


CONTINUOUS = [f for f in BUNDLE["fixtures"] + BUNDLE["readme"]
              if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"])
                      or f["model"].get("unrestricted"))
              and isinstance(f["model"].get("optimize"), str)]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _same(a, b):
    """Bit-for-bit equal, except that a NaN equals any NaN (its payload is not part of the contract)."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and np.array_equal(_bits(a)[~nan], _bits(b)[~nan])


def _cpu_model(jm):
    """The host Model of jm as Model.solve() leaves it before the upload (presolve applied), without a device tableau."""
    import jslpsolver_b200.tableau as T
    from jslpsolver_b200.model import Model, presolve
    saved = T.GpuTableau
    T.GpuTableau = lambda *a, **k: None
    try:
        m = Model().loadJson(jm)
    finally:
        T.GpuTableau = saved
    if m.usePresolve:
        m.presolveResult = presolve(m)
        for v in m.presolveResult.fixedVariables:
            v.cost = 0
    return m


def check_crash(M, vrow, vcol, enter, leave, engine, unres=None, simplex=True, check_cycles=True):
    """jslp_crash (+ simplex()) on the device against the oracle restatement from the same tableau, bit for bit."""
    from jslpsolver_b200 import _lib
    from jslpsolver_b200.tableau import GpuTableau
    from oracle import ref_model, warmstart as W
    g = GpuTableau(P)
    g.engine = engine
    g.options = {_lib.OPT_PIVOT_LOG_CAP: 1 << 20}
    g.upload(M, vrow, vcol, unres)
    o = ref_model.OracleTableau(M, vrow, vcol, precision=P, unrestricted=unres, check_cycles=check_cycles,
                                fast_cycles=True, pivot_log=1 << 20)
    recs, n = g.crash(enter, leave)
    orecs, on = W.crash(o, enter, leave, P)
    assert n == on
    assert np.array_equal(recs, orecs), (recs, orecs)
    assert _same(g.matrix2d(), o.matrix())
    gv, gc = g.varIndexByRow, g.varIndexByCol
    ov, oc = o.maps()
    assert np.array_equal(gv, ov) and np.array_equal(gc, oc)
    assert len(g.pivot_log()) == 0  # crash pivots are not simplex pivots
    if simplex:
        g.model = type("CycleCheck", (), {"checkForCycles": check_cycles})()
        g.simplex()
        st = g.lastStatus
        ost = o.simplex()
        assert (st.feasible, st.bounded, st.phase1_pivots, st.phase2_pivots) == \
               (ost.feasible, ost.bounded, ost.lastP1, ost.lastP2)
        assert _bits([st.evaluation]) == _bits([ost.evaluation]) or not st.feasible
        assert _same(g.matrix2d(), o.matrix())
        gv, gc = g.varIndexByRow, g.varIndexByCol
        ov, oc = o.maps()
        assert np.array_equal(gv, ov) and np.array_equal(gc, oc)
        glog, olog = g.pivot_log(), o.pivot_log()
        assert np.array_equal(glog, olog[len(olog) - len(glog):])
        assert len(glog) == st.phase1_pivots + st.phase2_pivots
    g.close()
    return recs, n, (st if simplex else None)


def _basis_of_fixture(jm):
    from oracle import ref_model, warmstart as W
    cold = ref_model.solve_full(jm, fast_cycles=True)
    if not (cold.feasible and cold.bounded):
        return None
    return W.basis(jm, cold)


@pytest.mark.parametrize("engine", ENGINES)
def test_fixtures_round_trip(engine):
    from jslpsolver_b200.warmstart import plan
    done = 0
    for f in CONTINUOUS:
        jm = strip_timeouts(f["model"])
        b = _basis_of_fixture(jm)
        if b is None:
            continue
        m = _cpu_model(jm)
        if m.presolveResult is not None and m.presolveResult.isInfeasible:
            continue
        it = m.initial_tableau()
        enter, leave, _ = plan(m, b)
        _, n, _ = check_crash(it.matrix, it.varIndexByRow, it.varIndexByCol, enter, leave, engine,
                           check_cycles=m.checkForCycles)
        assert n == len(b["variables"])
        done += 1
    assert done >= 10


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("kind", ["coef", "rhs", "cost", "add_rows", "add_vars", "del_rows", "del_vars", "rename",
                                  "infeasible", "unbounded"])
def test_seeded_edits(engine, kind):
    from jslpsolver_b200.warmstart import plan
    from test_warmstart_cpu import SEEDS, edit, mixed_model, _cold_basis
    for seed in SEEDS[:3]:
        jm = mixed_model(seed)
        b, _ = _cold_basis(jm)
        jm2 = edit(jm, kind, seed)
        m = _cpu_model(jm2)
        if m.presolveResult is not None and m.presolveResult.isInfeasible:
            continue
        it = m.initial_tableau()
        enter, leave, _ = plan(m, b)
        check_crash(it.matrix, it.varIndexByRow, it.varIndexByCol, enter, leave, engine, check_cycles=m.checkForCycles)


@pytest.mark.parametrize("engine", ENGINES)
def test_beyond_shared_memory(engine):
    """A 601 x 551 dense packing LP (beyond one CTA's shared memory) with 2 % coefficient noise, warm-started from the
    basis of the unperturbed LP."""
    from jslpsolver_b200 import problems
    from oracle import ref_model
    A, b, c = problems.dense_packing_lp_arrays(550, 600, 12345)
    it0 = problems.lp_tableau(A, b, c)
    o = ref_model.OracleTableau(it0.matrix, it0.varIndexByRow, it0.varIndexByCol, precision=P, fast_cycles=True)
    o.simplex()
    vrow, vcol = o.maps()
    n_var = len(c)
    var_labels = set(int(x) for x in it0.varIndexByCol[1:])
    enter = np.array([x for x in vrow[1:] if int(x) in var_labels], dtype=np.int32)
    leave = np.zeros(len(vrow) + len(vcol) - 2, dtype=np.uint8)
    leave[[int(x) for x in vcol[1:] if int(x) not in var_labels]] = 1
    rng = np.random.default_rng(12346)
    it = problems.lp_tableau(A * (1 + 0.02 * rng.standard_normal(A.shape)), b, c)
    recs, n, _ = check_crash(it.matrix, it.varIndexByRow, it.varIndexByCol, enter, leave, engine)
    assert n == len(enter) and n_var > n > 0


@pytest.mark.parametrize("engine", [0, 4])
def test_config3_from_stored_basis(engine):
    """Config 3 (2001 x 2001 dense packing) warm-started from the optimal vrow stored with its golden result: 65 crash
    pivots, then the oracle's simplex bit for bit, and the stored HiGHS objective to 1e-9."""
    import os
    from jslpsolver_b200 import problems
    from conftest import ROOT
    g = np.load(os.path.join(ROOT, "tests", "golden", "config3_dense2000.npz"))
    it = problems.dense_packing_lp_tableau(2000, 2000, 12345)
    var_labels = set(int(x) for x in it.varIndexByCol[1:])
    enter = np.array([x for x in g["vrow"][1:] if int(x) in var_labels], dtype=np.int32)
    leave = np.zeros(len(g["vrow"]) + len(g["vcol"]) - 2, dtype=np.uint8)
    leave[[int(x) for x in g["vcol"][1:] if int(x) not in var_labels]] = 1
    recs, n, st = check_crash(it.matrix, it.varIndexByRow, it.varIndexByCol, enter, leave, engine)
    assert n == 65 and st.feasible and st.bounded
    highs = float(g["highs_objective"])
    assert abs(abs(st.evaluation) - abs(highs)) <= 1e-9 * abs(highs)


# ---------------------------------------------------------------- geometry edges of k_crash_select
def _edge_tableau(H, W, seed):
    rng = np.random.default_rng(seed)
    M = rng.integers(-9, 10, size=(H, W)).astype(np.float64)
    M[1:, 0] = np.abs(M[1:, 0]) + 1.0
    vrow = np.concatenate([[-1], np.arange(W - 1, W - 1 + H - 1)]).astype(np.int32)  # slacks W-1 ..
    vcol = np.concatenate([[-1], np.arange(W - 1)]).astype(np.int32)                # structurals 0 .. W-2
    return M, vrow, vcol


@pytest.mark.parametrize("H", [4096, 4097, 4098])
@pytest.mark.parametrize("engine", [0, 2])
def test_rows_at_the_pass_edge(H, engine):
    M, vrow, vcol = _edge_tableau(H, 9, H)
    c = 1
    M[1:, c] = 1.0
    M[3, c], M[H - 1, c] = 7.5, -7.5             # a tie of opposite sign across passes: row 3 wins
    M[5, c] = np.nan                               # never eligible
    M[6, 2], M[7, 2], M[8, 2], M[9, 2] = P, -P, 0.0, -0.0  # at the threshold / signed zeros: not eligible
    M[1:, 2] = np.where((np.arange(1, H) > 9) | (np.arange(1, H) < 6), 0.0, M[1:, 2])  # untouched by pivot 1
    M[H - 1, 2] = -2.0 * P                         # the only eligible entry of column 2, in the last pass
    leave = np.ones(len(vrow) + len(vcol) - 2, dtype=np.uint8)
    enter = np.array([0, 1, 0], dtype=np.int32)   # the third entry is already basic
    recs, n, _ = check_crash(M, vrow, vcol, enter, leave, engine, simplex=False)
    assert recs[0, 1] == 3 and recs[1, 1] == H - 1 and recs[2, 3] == -2 and n == 2


@pytest.mark.parametrize("engine", [0, 1])
def test_empty_leave_mask_rejects_all(engine):
    M, vrow, vcol = _edge_tableau(50, 12, 3)
    leave = np.zeros(len(vrow) + len(vcol) - 2, dtype=np.uint8)
    recs, n, _ = check_crash(M, vrow, vcol, np.arange(11, dtype=np.int32), leave, engine)
    assert n == 0 and (recs[:, 3] == -1).all()


@pytest.mark.parametrize("engine", ENGINES)
def test_list_longer_than_one_graph(engine):
    """33 entries: one more than a graph holds; a mask that gives up only some rows, so some are rejected."""
    M, vrow, vcol = _edge_tableau(80, 40, 4)
    rng = np.random.default_rng(5)
    leave = np.zeros(len(vrow) + len(vcol) - 2, dtype=np.uint8)
    leave[rng.choice(np.arange(39, 39 + 79), size=30, replace=False)] = 1
    enter = rng.permutation(39)[:33].astype(np.int32)
    recs, n, _ = check_crash(M, vrow, vcol, enter, leave, engine)
    assert len(recs) == 33 and n > 0


# ---------------------------------------------------------------- the public interface
BERLIN = {"optimize": "capacity", "opType": "max",
          "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
          "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                        "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}


@pytest.mark.parametrize("engine", ENGINES)
def test_solve_with_basis_equals_oracle(engine):
    import json
    import jslpsolver_b200 as J
    from oracle import ref_model, warmstart as W
    s = J.Solver()
    s.engine = engine
    cold = s.Solve(BERLIN, full=True)
    b = cold.basis()
    assert json.loads(json.dumps(b)) == b
    for jm in (BERLIN, dict(BERLIN, constraints=dict(BERLIN["constraints"], plane={"max": 40}))):
        warm = s.Solve(jm, basis=b)
        osol, _, _, _ = W.warm_solve(jm, b)
        assert warm == ref_model.simplify(osol)
        full = s.Solve(jm, full=True, basis=b)
        ws = full.warmStart
        assert ws["pivots"] == len(ws["entered"]) and ws["rejected"] == [] and ws["alreadyBasic"] == []
        assert full.basis()["variables"]
    assert s.Solve(BERLIN) == ref_model.Solve(BERLIN)

"""Pins the oracle (oracle/) against every golden vector the reference holds for the LP/MIP
path: the `expects` blocks of the 47 test/test-sanity fixtures (compared exactly as
src/solver.integration.test.ts:60-100 does) and the README / integration-test known answers.
CPU only."""
import numpy as np
import pytest

from conftest import load_bundle
from helpers import compare_solutions, strip_timeouts
from oracle import ref_model

BUNDLE = load_bundle()


@pytest.mark.parametrize("fx", BUNDLE["fixtures"] + BUNDLE["readme"], ids=lambda f: f["file"])
def test_fixture_expects(fx):
    res = ref_model.Solve(strip_timeouts(fx["model"]), fast_cycles=True)
    bad = compare_solutions(res, fx["expects"])
    assert not bad, bad     # every fixture on every listed key, no exceptions


def test_readme_berlin_pivot_sequence():
    """SURVEY.md appendix A worked example: pivots (2,2) then (1,1), exact tie on row 1."""
    fx = [f for f in BUNDLE["readme"] if f["file"] == "README Berlin Airlift"][0]
    sol = ref_model.solve_full(fx["model"], pivot_log=16)
    log = sol.tableau.pivot_log()
    assert log[:, :2].tolist() == [[2, 2], [1, 1]]
    vrow, vcol = sol.tableau.maps()
    assert vrow.tolist() == [-1, 3, 4, 2] and vcol.tolist() == [-1, 0, 1]
    assert sol.tableau.matrix()[0, 0] == -1080000


def test_cycle_detectors_agree():
    """cycles_fast is only valid under the calling discipline of simplex.ts (checked after
    every push, stop at first hit); under that discipline it must equal the literal scan."""
    import ctypes
    L = ref_model.lib()
    rng = np.random.default_rng(7)
    for trial in range(300):
        n_sym = int(rng.integers(1, 5))
        seq = rng.integers(0, n_sym, size=(40, 2)).astype(np.int32)
        for n in range(1, len(seq) + 1):
            cur = np.ascontiguousarray(seq[:n])
            s1, l1, s2, l2 = (ctypes.c_long() for _ in range(4))
            h1 = L.orc_cycles_ref(cur.ctypes.data, n, ctypes.byref(s1), ctypes.byref(l1))
            h2 = L.orc_cycles_fast(cur.ctypes.data, n, ctypes.byref(s2), ctypes.byref(l2))
            assert h1 == h2, (trial, n)
            if h1:
                assert (s1.value, l1.value) == (s2.value, l2.value)
                break


def test_js_semantics_helpers():
    assert ref_model.js_keys({"b": 1, "21": 1, "a": 1, "3": 1, "03": 1}) == ["3", "21", "b", "a", "03"]
    assert ref_model.js_round(2.5) == 3 and ref_model.js_round(-2.5) == -2
    assert ref_model.js_round(0.49999999999999994) == 0


def test_cut_rows_known_answers():
    """addCutConstraints RHS rule (cutting-strategies.ts:36-62; the reference pins the same
    values in cutting-strategies.test.ts:73-101): basic var at value 2.5, cut x >= 3 -> RHS
    -(3-2.5) = -0.5; cut x <= 2 -> RHS 2-2.5 = -0.5; non-basic var -> RHS sign*value."""
    M = np.array([[0.0, 1.0, 2.0], [2.5, 0.5, -1.0], [4.0, 1.0, 1.0]])
    vrow = np.array([-1, 2, 3], dtype=np.int32)   # var 2 basic in row 1
    vcol = np.array([-1, 0, 1], dtype=np.int32)   # vars 0, 1 non-basic
    t = ref_model.OracleTableau(M, vrow, vcol)
    t.add_cuts([("min", 2, 3.0), ("max", 2, 2.0), ("min", 0, 1.0), ("max", 1, 7.0)])
    X = t.matrix()
    assert X.shape == (7, 3)
    assert X[3].tolist() == [-0.5, 0.5, -1.0]
    assert X[4].tolist() == [-0.5, -0.5, 1.0]
    assert X[5].tolist() == [-1.0, -1.0, 0.0]
    assert X[6].tolist() == [7.0, 0.0, 1.0]
    vrow2, _ = t.maps()
    assert vrow2.tolist() == [-1, 2, 3, 4, 5, 6, 7]


def _mip_tableau(rhs, basic_vars, integers, precision=1e-9):
    """Tableau whose row r >= 1 holds variable basic_vars[r-1] at value rhs[r-1] (RHS = column 0, as in the
    reference's real tableau; its unit tests put it in column 2 of a mock)."""
    H = len(rhs) + 1
    M = np.zeros((H, 3))
    M[1:, 0] = rhs
    vrow = np.array([-1] + list(basic_vars), dtype=np.int32)
    n_vars = 3 + H - 2  # the oracle sizes its inverse maps by width + height - 2, like the reference
    free = [v for v in range(n_vars) if v not in basic_vars]
    assert len(free) == 2
    vcol = np.array([-1] + free, dtype=np.int32)
    return ref_model.OracleTableau(M, vrow, vcol, precision=precision, integers=list(integers))


def test_is_integral_known_answers():
    """The cases of the reference's mip-utils.test.ts:173-300 (isIntegral, mip-utils.ts:43-61)."""
    assert _mip_tableau([5.0, 3.0], [1, 2], [1, 2]).is_integral() is True
    assert _mip_tableau([5.0, 3.7], [1, 2], [1, 2]).is_integral() is False
    assert _mip_tableau([5.5], [1], []).is_integral() is True                 # no integer variables
    assert _mip_tableau([5.0], [1], [1, 2]).is_integral() is True             # variable 2 is not basic
    assert _mip_tableau([4.9999999], [1], [1], precision=1e-6).is_integral() is True


def test_most_fractional_known_answers():
    """The cases of mip-utils.test.ts:431-565 (getMostFractionalVar, mip-utils.ts:100-126): largest distance
    to the nearest integer, the first integer variable wins ties, non-basic variables are skipped."""
    assert _mip_tableau([5.3, 3.7], [1, 2], [1, 2]).most_fractional() == (1, 5.3)   # both 0.3 away: first wins
    assert _mip_tableau([5.1, 3.5], [1, 2], [1, 2]).most_fractional() == (2, 3.5)
    assert _mip_tableau([5.3], [1], [1, 2]).most_fractional()[0] == 1               # variable 2 not basic
    i, v = _mip_tableau([5.0], [1], [1]).most_fractional()                          # nothing fractional
    assert i < 0 and v == 0.0
    i, _ = _mip_tableau([5.5], [1], []).most_fractional()                           # no integer variables
    assert i < 0


def test_solver_options_known_answers():
    """Known answers of the reference's solver.options.test.ts:68-136 that run through the default
    branch-and-cut service (timeout removed: it is wall-clock)."""
    r = ref_model.simplify(ref_model.solve_full({
        "optimize": "profit", "opType": "max", "constraints": {"capacity": {"max": 10}},
        "variables": {"x": {"profit": 5, "capacity": 2}}, "ints": {"x": 1}}))
    assert r["feasible"] is True and r["x"] == 5
    r = ref_model.simplify(ref_model.solve_full({
        "optimize": "profit", "opType": "max", "constraints": {"budget": {"max": 100}},
        "variables": {"a": {"profit": 10, "budget": 10}, "b": {"profit": 15, "budget": 15}, "c": {"profit": 20, "budget": 20}},
        "ints": {"a": 1, "b": 1, "c": 1}, "tolerance": 0.1}))
    assert r["feasible"] is True and r["result"] >= 90
    r = ref_model.simplify(ref_model.solve_full({
        "optimize": "profit", "opType": "max", "constraints": {"budget": {"max": 100}},
        "variables": {"a": {"profit": 10, "budget": 10}, "b": {"profit": 8, "budget": 10}},
        "ints": {"a": 1, "b": 1}, "tolerance": 0}))
    assert r["feasible"] is True and r["result"] == 100


# ------------------------------------------------------------------ useMIRCuts (cutting-strategies.ts:74-212, branch-and-cut.ts:38-51)
def _mir_tableau():
    """The mock of cutting-strategies.test.ts:185-199: width 4, height 3, row 1 basic variable integer with right-hand
    side 5.3, column variables y (integer) and z (continuous)."""
    M = np.zeros((3, 4))
    M[1] = [5.3, 2.5, -1.5, 0.25]
    M[2] = [4.0, 1.0, 1.0, 1.0]
    vrow = np.array([-1, 1, 0], dtype=np.int32)
    vcol = np.array([-1, 2, 3, 4], dtype=np.int32)
    return ref_model.OracleTableau(M, vrow, vcol, precision=1e-9, integers=[1, 2])


def test_mir_cut_known_answers():
    """The reference's own unit tests pin structure only (cutting-strategies.test.ts:145-330): false on the cost row, on a
    non-integer or undefined basic variable, on an integral or near-integral right-hand side; true + one more row on a
    fractional one.  The coefficient formulas are checked here against a direct evaluation of cutting-strategies.ts:116-131
    and 174-193."""
    import math
    t = _mir_tableau()
    assert not t.add_mir_cut(0) and not t.add_mir_cut(0, upper=True)          # cost row
    assert not t.add_mir_cut(2) and not t.add_mir_cut(2, upper=True)          # basic variable 0 is not integer
    t2 = _mir_tableau()
    X = t2.matrix(); X[1, 0] = 5.0
    t2 = ref_model.OracleTableau(X, *t2.maps(), precision=1e-9, integers=[1, 2])
    assert not t2.add_mir_cut(1)                                              # integral right-hand side
    X[1, 0] = 5.0000001
    t3 = ref_model.OracleTableau(X, np.array([-1, 1, 0], dtype=np.int32), np.array([-1, 2, 3, 4], dtype=np.int32),
                                 precision=1e-6, integers=[1, 2])
    assert not t3.add_mir_cut(1)                                              # near-integral counts as integral
    assert t.add_mir_cut(1)
    Y = t.matrix()
    assert Y.shape == (4, 4) and t.maps()[0][3] == 5                          # new slack takes the next element index
    f = 5.3 - math.floor(5.3)
    want = [math.floor(5.3) - 5.3,
            (math.floor(2.5) + max(0, 2.5 - math.floor(2.5) - f) / (1 - f)) - 2.5,   # y is integer
            min(0, -1.5 / (1 - f)) - (-1.5),                                           # z is continuous
            min(0, 0.25 / (1 - f)) - 0.25]                                             # var 4: undefined -> continuous rule
    assert Y[3].tolist() == want
    assert t.add_mir_cut(1, upper=True)
    Z = t.matrix()
    tc = 2.5 - math.floor(2.5)
    assert Z[4].tolist() == [-f, (-(1 - tc) * f) / tc, (-1.5 * f) / (1 - f), -0.25]
    assert t.fractional_volume(False) == 0 or t.fractional_volume(True) >= 0


def test_mir_cuts_are_valid_inequalities():
    """Mixed-integer rounding cuts cut off no integer point: with options.useMIRCuts every MIP fixture keeps its optimum
    (the reference's options test only asks for feasible && result > 0, solver.options.test.ts:252-272)."""
    model = {"optimize": "profit", "opType": "max", "constraints": {"resource": {"max": 100}},
             "variables": {"x": {"profit": 10, "resource": 7}, "y": {"profit": 15, "resource": 11}},
             "ints": {"x": 1, "y": 1}, "options": {"useMIRCuts": True}}
    res = ref_model.Solve(model)
    assert res["feasible"] and res["result"] > 0 and res["result"] == ref_model.Solve(dict(model, options={}))["result"]
    for fx in BUNDLE["fixtures"]:
        m = strip_timeouts(fx["model"])
        if not (m.get("ints") or m.get("binaries")) or m.get("tolerance") or (m.get("options") or {}).get("tolerance"):
            continue  # a tolerance accepts any incumbent within it: the path, hence the answer, may differ
        m["options"] = dict(m.get("options") or {}, useMIRCuts=True)
        r = ref_model.Solve(m, fast_cycles=True)
        bad = [b for b in compare_solutions(r, fx["expects"]) if b.startswith(("result", "feasible"))]
        assert not bad, (fx["file"], bad)


# ------------------------------------------------------------------ dynamic-modification.ts:16-316
def _dm_tableau(M, vrow, vcol, opt=None, precision=1e-9):
    return ref_model.OracleTableau(np.array(M, dtype=np.float64), np.array(vrow, dtype=np.int32), np.array(vcol, dtype=np.int32),
                                   precision=precision, opt_rc=None if opt is None else np.array(opt, dtype=np.float64))


def test_dynamic_modification_known_answers():
    """The numeric known answers of the reference's dynamic-modification.test.ts, on tableaux laid out like its mock
    (width 4, height 3; rows labelled 0..2 with row 0 = cost row, columns labelled 3..5)."""
    base = [[10.0, 1, 2, 3], [20.0, 4, 5, 6], [30.0, 7, 8, 9]]
    # updateRightHandSide, constraint in the basis (:183-191): matrix[1*4+0] = 10 -> 7
    t = _dm_tableau([[0.0, 0, 0, 0], [10.0, 0, 0, 0], [0.0, 0, 0, 0]], [-1, 1, 2], [-1, 3, 4, 5])
    t.update_rhs(1, 3)
    assert t.matrix()[1, 0] == 7
    # constraint not in the basis (:194-211): every row, rhs -= 1 * column entry
    t = _dm_tableau([[10.0, 2, 0, 0], [20.0, 3, 0, 0], [30.0, 4, 0, 0]], [-1, 1, 2], [-1, 3, 4, 5], opt=[[10.0, 5, 0, 0]])
    t.update_rhs(3, 1)
    assert t.matrix()[:, 0].tolist() == [8, 17, 26] and t.optional()[0, 0] == 5
    # updateConstraintCoefficient (:229-268)
    t = _dm_tableau(base, [-1, 1, 2], [-1, 3, 4, 5])
    with pytest.raises(ValueError):
        t.update_coefficient(1, 1, 1.0)
    m0 = t.matrix()
    t.update_coefficient(1, 4, 3)            # variable 4 non-basic in column 2: entry -= 3
    assert t.matrix()[1, 2] == m0[1, 2] - 3
    t.update_coefficient(1, 2, 2)            # variable 2 basic in row 2: row 1 += 2 * row 2
    assert t.matrix()[1].tolist() == [20 + 60, 4 + 14, (5 - 3) + 16, 6 + 18]
    # updateCost (:273-312)
    t = _dm_tableau(base, [-1, 1, 2], [-1, 3, 4, 5], opt=[[1.0, 1, 1, 1]])
    t.update_cost(4, 5)                      # non-basic, column 2: row 0 entry -= 5
    assert t.matrix()[0, 2] == 2 - 5
    t.update_cost(1, 3)                      # basic in row 1: cost row += 3 * row 1
    assert t.matrix()[0].tolist() == [10 + 60, 1 + 12, -3 + 15, 3 + 18]
    t.update_cost(2, 3, opt_slot=0)          # priority > 0: optional objective += 3 * row 2
    assert t.optional()[0].tolist() == [1 + 90, 1 + 21, 1 + 24, 1 + 27]
    # addConstraint (:317-412): new row, sign, terms of non-basic and basic variables, maps
    t = _dm_tableau(base, [-1, 1, 2], [-1, 3, 4, 5])
    t.add_constraint(True, 5, 10, [])
    assert t.state().height == 4 and t.matrix()[3].tolist() == [5, 0, 0, 0] and t.maps()[0][3] == 10 and t.row_of(10) == 3
    t.add_constraint(False, 5, 11, [(3, 3.0)])
    assert t.matrix()[4].tolist() == [-5, -3, 0, 0]
    t.add_constraint(True, 10, 12, [(1, 2.0)])   # variable 1 basic in row 1: row -= 2 * row 1
    assert t.matrix()[5].tolist() == [10 - 2 * 20, -8, -10, -12]
    # removeConstraint (:417-461): swap with the last row
    t = _dm_tableau(base, [-1, 1, 2], [-1, 3, 4, 5])
    t.remove_constraint(1)
    assert t.state().height == 2 and t.matrix()[1].tolist() == [30, 7, 8, 9] and t.maps()[0][1] == 2 and t.row_of(1) == -1
    # addVariable (:464-529): one more column, cost entry in row 0, maps
    t = _dm_tableau(base, [-1, 1, 2], [-1, 3, 4, 5])
    t.add_variable(10, -5.0)
    X = t.matrix()
    assert X.shape == (3, 5) and X[0].tolist() == [10, 1, 2, 3, -5] and X[1].tolist() == [20, 4, 5, 6, 0] and t.maps()[1][4] == 10
    # putInBase / takeOutOfBase (:84-141): first row / column with a non-zero entry, then pivot
    t = _dm_tableau([[0.0, 0, 0, 0], [1.0, 0, 2, 0], [1.0, 5, 3, 0]], [-1, 1, 2], [-1, 3, 4, 5], precision=1e-9)
    assert t.put_in_base(1) == 1 and t.put_in_base(3) == 2 and t.maps()[0][2] == 3
    assert t.take_out_of_base(4) == 2 and t.take_out_of_base(1) == 2   # row 1's first non-zero column is 2


# ------------------------------------------------------------------ enhanced service (enhanced-branch-and-cut.ts)
def test_enhanced_service_known_answers():
    """solver.options.test.ts:139-250: every nodeSelection / branching choice is feasible, and all node-selection
    strategies reach the same optimum; on the MIP fixtures without a tolerance every combination keeps the optimum."""
    base = {"optimize": "profit", "opType": "max", "constraints": {"capacity": {"max": 50}, "labor": {"max": 40}},
            "variables": {"table": {"profit": 12, "capacity": 3, "labor": 5}, "chair": {"profit": 8, "capacity": 2, "labor": 3}},
            "ints": {"table": 1, "chair": 1}}
    results = [ref_model.Solve(dict(base, options={"nodeSelection": ns})) for ns in ("best-first", "depth-first", "hybrid")]
    assert all(r["feasible"] and r["result"] > 0 for r in results)
    assert results[0]["result"] == results[1]["result"] == results[2]["result"] == ref_model.Solve(base)["result"]
    knap = {"optimize": "value", "opType": "max", "constraints": {"weight": {"max": 100}},
            "variables": {"item1": {"value": 60, "weight": 10}, "item2": {"value": 100, "weight": 20}, "item3": {"value": 120, "weight": 30}},
            "ints": {"item1": 1, "item2": 1, "item3": 1}}
    for br in ("most-fractional", "pseudocost", "strong"):
        assert ref_model.Solve(dict(knap, options={"branching": br}))["feasible"]
    for fx in BUNDLE["fixtures"]:
        m = strip_timeouts(fx["model"])
        if not (m.get("ints") or m.get("binaries")) or m.get("tolerance") or (m.get("options") or {}).get("tolerance"):
            continue
        for opts in ({"nodeSelection": "hybrid"}, {"nodeSelection": "depth-first", "branching": "strong"}, {"branching": "most-fractional"},
                     {"useIncremental": True}, {"useIncremental": True, "nodeSelection": "depth-first"}):
            r = ref_model.Solve(dict(m, options=dict(m.get("options") or {}, **opts)), fast_cycles=True)
            bad = [b for b in compare_solutions(r, fx["expects"]) if b.startswith(("result", "feasible"))]
            assert not bad, (fx["file"], opts, bad)


# ------------------------------------------------------------------ independent cross-check (not the reference, not the oracle)
def _random_model(rng, n, m, integer):
    cons = {f"c{i}": ({"max": float(rng.integers(20, 200))} if rng.random() < 0.75 else {"min": float(rng.integers(1, 15))}) for i in range(m)}
    vars_ = {}
    for j in range(n):
        v = {"obj": float(rng.integers(1, 40))}
        for i in range(m):
            if rng.random() < 0.7:
                v[f"c{i}"] = float(rng.integers(1, 12))
        vars_[f"x{j}"] = v
    model = {"optimize": "obj", "opType": "max", "constraints": cons, "variables": vars_}
    if integer:
        model["ints"] = {f"x{j}": 1 for j in range(n) if rng.random() < 0.6}
    return model


def _scipy_solve(model):
    from scipy.optimize import Bounds, LinearConstraint, milp
    names = list(model["variables"])
    c = -np.array([model["variables"][v].get("obj", 0.0) for v in names])   # milp minimises
    rows, lo, hi = [], [], []
    for cname, spec in model["constraints"].items():
        rows.append([model["variables"][v].get(cname, 0.0) for v in names])
        lo.append(spec.get("min", -np.inf))
        hi.append(spec.get("max", np.inf))
    integrality = np.array([1 if v in model.get("ints", {}) else 0 for v in names])
    res = milp(c, constraints=LinearConstraint(np.array(rows), lo, hi), integrality=integrality, bounds=Bounds(0, np.inf))
    return (res.status == 0), (-res.fun if res.status == 0 else None), res.status


def test_oracle_optimum_equals_an_independent_solver():
    """The oracle is pinned on the reference's own golden vectors; this adds a check against a solver that shares no code
    or rule with either: SciPy's HiGHS (`scipy.optimize.milp`) on random bounded LPs and small MIPs -- same
    feasibility verdict, objective within 1e-7 relative (different algorithms, so optimal VERTICES may differ)."""
    pytest.importorskip("scipy")
    rng = np.random.default_rng(2024)
    checked = 0
    for k in range(60):
        integer = k % 2 == 1
        model = _random_model(rng, int(rng.integers(3, 9)), int(rng.integers(2, 7)), integer)
        ok, val, status = _scipy_solve(model)
        if status not in (0, 2):      # unbounded etc.: skip, the generator makes those rare
            continue
        res = ref_model.Solve(model, fast_cycles=True)
        assert bool(res["feasible"]) == ok, (k, res, status)
        if ok:
            assert res["bounded"] and abs(res["result"] - val) <= 1e-7 * max(1.0, abs(val)), (k, res["result"], val)
            checked += 1
    assert checked >= 30


def test_big_config_fixtures_agree_with_an_independent_solver():
    """The oracle's cached optimum of BASELINE config 3 (dense 2000x2000) and of the config-5 root relaxation equals the
    objective SciPy's HiGHS finds for the same arrays (tests/golden/make_big_golden.py stores both) to 1e-9 relative."""
    import os
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    z3 = np.load(os.path.join(gold, "config3_dense2000.npz"))
    z5 = np.load(os.path.join(gold, "config5_knapsack.npz"))
    for ours, highs in ((-float(z3["evaluation"][0]), float(z3["highs_objective"])),
                        (-float(z5["root_evaluation"][0]), float(z5["root_highs_objective"]))):
        assert abs(ours - highs) <= 1e-9 * abs(highs), (ours, highs)


def _random_model_mixed(rng, n, m, integer):
    """min / max / equal rows, max or min objective, costs of either sign: optimal, infeasible and unbounded instances."""
    cons = {}
    for i in range(m):
        r = rng.random()
        cons[f"c{i}"] = ({"max": float(rng.integers(5, 60))} if r < 0.5 else
                         ({"min": float(rng.integers(5, 80))} if r < 0.85 else {"equal": float(rng.integers(5, 40))}))
    vars_ = {}
    for j in range(n):
        v = {"obj": float(rng.integers(-10, 40))}
        for i in range(m):
            if rng.random() < 0.6:
                v[f"c{i}"] = float(rng.integers(1, 12))
        vars_[f"x{j}"] = v
    model = {"optimize": "obj", "opType": "max" if rng.random() < 0.7 else "min", "constraints": cons, "variables": vars_}
    if integer:
        model["ints"] = {f"x{j}": 1 for j in range(n) if rng.random() < 0.5}
    return model


def _scipy_solve_mixed(model):
    from scipy.optimize import Bounds, LinearConstraint, milp
    names = list(model["variables"])
    sign = -1.0 if model["opType"] == "max" else 1.0
    c = sign * np.array([model["variables"][v].get("obj", 0.0) for v in names])
    rows, lo, hi = [], [], []
    for cname, spec in model["constraints"].items():
        rows.append([model["variables"][v].get(cname, 0.0) for v in names])
        if "equal" in spec:
            lo.append(spec["equal"]); hi.append(spec["equal"])
        else:
            lo.append(spec.get("min", -np.inf)); hi.append(spec.get("max", np.inf))
    integrality = np.array([1 if v in model.get("ints", {}) else 0 for v in names])
    res = milp(c, constraints=LinearConstraint(np.array(rows), lo, hi), integrality=integrality, bounds=Bounds(0, np.inf))
    return res.status, (sign * res.fun if res.status == 0 else None)


def test_oracle_verdicts_equal_an_independent_solver_on_mixed_models():
    """Optimal / infeasible / unbounded verdicts and optimal values against SciPy's HiGHS on models with `min`, `max` and
    `equal` rows, both objective senses, costs of either sign, LPs and MIPs (HiGHS status 0 / 2 / 3)."""
    pytest.importorskip("scipy")
    rng = np.random.default_rng(5)
    seen = {0: 0, 2: 0, 3: 0}
    for k in range(200):
        model = _random_model_mixed(rng, int(rng.integers(3, 14)), int(rng.integers(2, 9)), k % 3 == 1)
        status, val = _scipy_solve_mixed(model)
        res = ref_model.Solve(model, fast_cycles=True)
        if status == 0:
            assert res["feasible"] and res["bounded"] and abs(res["result"] - val) <= 1e-7 * max(1.0, abs(val)), (k, res, val)
        elif status == 2:
            assert not res["feasible"], (k, res)
        elif status == 3:
            assert not (res["feasible"] and res["bounded"]), (k, res)
        seen[status] = seen.get(status, 0) + 1
    assert seen[0] >= 40 and seen[2] >= 40 and seen[3] >= 15, seen


def test_oracle_root_tableau_is_the_front_ends_bit_for_bit():
    """Tableau.setModel (tableau.ts:332-378) in the oracle and in the front end: every fixture's root tableau has the
    same bits, signed zeros included (JS stores -1 * 0 and -(0) as -0 in the cost row and in `min` rows)."""
    from jslpsolver_b200.model import Model
    from oracle.ref_model import RefModel
    for fx in load_bundle()["fixtures"]:
        jm = strip_timeouts(fx["model"])
        a = Model().loadJson(jm).initial_tableau().matrix
        b = RefModel(None).loadJson(jm).build_tableau()[0]
        assert a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64)), fx["file"]

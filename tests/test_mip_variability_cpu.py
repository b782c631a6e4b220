"""Near-optimal variability of a MIP (DESIGN.md section 2o) without a GPU: the restatement of
tests/mip_variability_oracle.py against SciPy's HiGHS (every range end a MIP of its own) and against brute force, the
Sudoku check of rule 2, witnesses, width invariance, unbounded ends, the node limit, Variability()'s refusals and the
jslp_target_batch declaration against its ctypes mirror."""
from __future__ import annotations

import math

import numpy as np
import pytest

import mip_variability_oracle as MO
from jslpsolver_b200 import problems
from jslpsolver_b200.model import Model
from test_pool_cpu import _types, enumerable_random_mips, enumerate_all, fixture

SMALL = ["Integer Berlin Air Lift Problem.json", "Integer Chocolate Problem.json", "Integer Clothing Shop Problem.json",
         "Integer Clothing Shop Problem II.json", "Integer Sports Complex Problem.json", "Integer Wood Problem.json",
         "Integer Wood Shop Problem.json", "Cutting stock.json", "TacoParty.json", "Knapsack 1.json",
         "integration widget"]


@pytest.fixture(scope="module", autouse=True)
def _oracle_lib():
    from oracle import ref_model
    ref_model.build_oracle()


def random_mixed_mips(n: int) -> list:
    """The first n seeded random MIPs (6 variables, 4 rows, about half of them integer) whose relaxation is bounded and
    feasible and which have an integer plan."""
    from scipy.optimize import linprog
    from test_pool_cpu import arrays
    found = []
    for seed in range(200):
        jm = problems.random_mip_model(6, 4, seed=seed, integer_fraction=0.5)
        if not jm.get("ints"):
            continue
        names, _, c, A, b, upper = arrays(jm)
        if linprog(c, A_ub=A, b_ub=b, bounds=[(0, u) for u in upper], method="highs").status != 0:
            continue
        if highs(jm, None, 0, None)[0] != 0:
            continue
        found.append(jm)
        if len(found) == n:
            break
    return found


# ---- HiGHS ------------------------------------------------------------------------------------------------------
def lp_data(jm: dict):
    """(model, objective c over model.variables, rows [(constraint, a)], integrality) of the model as loadJson reads
    it: every row of m.constraints, the binaries' `x <= 1` rows included."""
    m = Model().loadJson(jm)
    pos = {v.index: j for j, v in enumerate(m.variables)}
    c = np.array([float(v.cost) for v in m.variables])
    rows = []
    for con in m.constraints:
        a = np.zeros(len(m.variables))
        for t in con.coef.values():
            a[pos[t.variable.index]] += t.coefficient
        rows.append((con, a))
    return m, c, rows, np.array([1 if v.isInteger else 0 for v in m.variables])


def highs(jm: dict, objective, sense: int, cap):
    """(status, value) of optimising objective (a vector over the variables, or None for the model's own objective)
    with sense -1 min / +1 max over the integer plans of jm, with the objective bound cap = (c, limit, is_min) when
    given.  status: 0 optimal, 2 infeasible, 3 unbounded, as scipy.optimize.milp reports them."""
    from scipy.optimize import Bounds, LinearConstraint, milp
    m, c, rows, integrality = lp_data(jm)
    A = np.array([a for _, a in rows])
    lo = np.array([-np.inf if con.isUpperBound else con.rhs for con, _ in rows])
    hi = np.array([con.rhs if con.isUpperBound else np.inf for con, _ in rows])
    cons = [LinearConstraint(A, lo, hi)]
    if cap is not None:
        cvec, limit, is_min = cap
        cons.append(LinearConstraint(cvec[None, :], -np.inf if is_min else limit, limit if is_min else np.inf))
    if objective is None:
        objective, sense = c, (-1 if m.isMinimization else 1)
    for presolve in (True, False):  # HiGHS's presolve reports "infeasible or unbounded" (4) where its solve tells
        res = milp(-sense * objective, constraints=cons, integrality=integrality, bounds=Bounds(0, np.inf),
                   options={"mip_rel_gap": 0, "presolve": presolve})
        if res.status != 4:
            break
    return res.status, (None if res.status != 0 else -sense * res.fun)


def highs_ranges(jm: dict, z_star: float, t: float):
    """{("v", id) / ("c", row position): (min, max)} of every variable and row slack by HiGHS."""
    m, c, rows, _ = lp_data(jm)
    scale = max(1.0, abs(z_star))
    cap = (c, z_star + t + 1e-9 * scale if m.isMinimization else z_star - t - 1e-9 * scale, m.isMinimization)
    out = {}
    targets = [(("v", v.id), np.eye(len(m.variables))[j], 0.0) for j, v in enumerate(m.variables)]
    for i, (con, a) in enumerate(rows):  # slack = rhs - a.x (max rows) or a.x - rhs (min rows)
        targets.append((("c", i), -a if con.isUpperBound else a, con.rhs if con.isUpperBound else -con.rhs))
    for key, vec, const in targets:
        ends = []
        for s in (-1, 1):
            st, val = highs(jm, vec, s, cap)
            ends.append(s * math.inf if st == 3 else None if st != 0 else val + const)
        out[key] = tuple(ends)
    return out


def same_ranges(got: dict, jm: dict, rel=1e-7):
    want = highs_ranges(jm, got["optimum"], got["allowance"])
    have = {("v", vid): (e["min"], e["max"]) for vid, e in got["variables"].items()}
    have.update({("c", i): (c["slack"]["min"], c["slack"]["max"]) for i, c in enumerate(got["constraints"])})
    # relative to the data: HiGHS meets rows and the objective bound within its own feasibility tolerance, which lets
    # an end over a single optimal point move by that much
    _, _, rows, _ = lp_data(jm)
    scale = max([1.0, abs(got["optimum"])] + [abs(con.rhs) for con, _ in rows] +
                [abs(x) for pair in want.values() for x in pair if x is not None and math.isfinite(x)])
    for key, (lo, hi) in want.items():
        for mine, theirs in zip(have[key], (lo, hi)):
            assert mine is not None and theirs is not None, (key, have[key], (lo, hi))
            if math.isinf(theirs):
                assert mine == theirs, (key, have[key], (lo, hi))
            else:
                assert abs(mine - theirs) <= rel * scale, (key, have[key], (lo, hi))


@pytest.mark.parametrize("name", SMALL)
@pytest.mark.parametrize("gap, absolute_gap", [(0.0, 0.0), (0.05, 0.0), (0.0, 3.0)])
def test_restatement_matches_highs_on_the_bundle(name, gap, absolute_gap):
    jm = fixture(name)
    got = MO.variability(jm, gap=gap, absolute_gap=absolute_gap, width=4)
    assert got["exact"]
    z_star = highs(jm, None, 0, None)[1]
    assert got["optimum"] == pytest.approx(z_star, rel=1e-9, abs=1e-9)
    same_ranges(got, jm)


@pytest.mark.parametrize("jm", random_mixed_mips(6), ids=lambda m: m["name"])
@pytest.mark.parametrize("gap, absolute_gap", [(0.0, 0.0), (0.05, 0.0), (0.0, 5.0)])
def test_restatement_matches_highs_on_random_mixed_mips(jm, gap, absolute_gap):
    got = MO.variability(jm, gap=gap, absolute_gap=absolute_gap, width=3)
    assert got["exact"]
    same_ranges(got, jm)


# ---- brute force --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jm", enumerable_random_mips(4), ids=lambda m: m["name"])
@pytest.mark.parametrize("absolute_gap", [0.0, 10.0, 1e4])
def test_restatement_matches_brute_force(jm, absolute_gap):
    brute = enumerate_all(jm)
    got = MO.variability(jm, absolute_gap=absolute_gap, width=2)
    sign = -1.0 if jm.get("opType") == "max" else 1.0
    f_star = brute[0][0]
    assert got["optimum"] == pytest.approx(sign * f_star, rel=1e-9, abs=1e-9)
    inside = [z for f, z in brute if f <= f_star + got["allowance"] + 1e-7 * max(1.0, abs(f_star))]
    for v in brute[0][1]:
        e = got["variables"][v]
        assert (round(e["min"]), round(e["max"])) == (min(z[v] for z in inside), max(z[v] for z in inside))
        assert abs(e["min"] - round(e["min"])) < 1e-7 and abs(e["max"] - round(e["max"])) < 1e-7


# ---- Sudoku: rule 2 -------------------------------------------------------------------------------------------------
def test_sudoku_every_binary_ranges_over_zero_and_one():
    got = MO.variability(fixture("Sudoku4x4.json"), width=8)
    assert got["exact"] and not got["unique"] and got["allowance"] == 0.0
    for vid, e in got["variables"].items():
        assert abs(e["min"]) < 1e-9 and abs(e["max"] - 1.0) < 1e-9, (vid, e)


def test_sudoku_givens_fix_their_cells():
    jm = fixture("Sudoku4x4.json")
    givens = ["x111", "x222", "x333", "x444", "x124"]
    jm = dict(jm, constraints=dict(jm["constraints"]), variables={k: dict(v) for k, v in jm["variables"].items()})
    for g in givens:
        jm["constraints"]["given_" + g] = {"min": 1}
        jm["variables"][g]["given_" + g] = 1
    got = MO.variability(jm, width=8)
    assert got["exact"]
    for g in givens:
        r, c = g[1], g[2]
        for v in range(1, 5):
            e = got["variables"][f"x{r}{c}{v}"]
            want = 1.0 if f"x{r}{c}{v}" == g else 0.0
            assert abs(e["min"] - want) < 1e-9 and abs(e["max"] - want) < 1e-9, (g, v, e)


# ---- witnesses and width --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name, gap", [("Integer Sports Complex Problem.json", 0.05), ("Knapsack 1.json", 0.01),
                                       ("Integer Clothing Shop Problem II.json", 0.1)])
def test_witnesses_are_integer_plans_within_the_allowance(name, gap):
    jm = fixture(name)
    got = MO.variability(jm, gap=gap, points=True, width=4)
    m, c, rows, integrality = lp_data(jm)
    ids = [v.id for v in m.variables]
    P = m.precision
    z_star, t = got["optimum"], got["allowance"]
    for vid, e in got["variables"].items():
        for side in ("min", "max"):
            w = e["arg" + side]
            x = np.array([w[i] for i in ids])
            assert np.all(np.abs(x[integrality == 1] - np.round(x[integrality == 1])) <= 1e-7), (vid, side)
            assert np.all(x >= -P)
            for con, a in rows:
                act = float(a @ x)
                assert (act <= con.rhs + 1e-7 if con.isUpperBound else act >= con.rhs - 1e-7), (vid, side, con.name)
            z = float(c @ x)
            assert (z <= z_star + t + 1e-7 if m.isMinimization else z >= z_star - t - 1e-7), (vid, side, z)
            assert w[vid] == e[side]


@pytest.mark.parametrize("name", ["Integer Sports Complex Problem.json", "Knapsack 1.json", "Sudoku4x4.json"])
def test_width_changes_no_range(name):
    jm = fixture(name)
    runs = [MO.variability(jm, gap=0.02, width=1), MO.variability(jm, gap=0.02, wave=256),
            MO.variability(jm, gap=0.02, width=64)]
    strip = lambda r: ({k: (e["min"], e["max"]) for k, e in r["variables"].items()},  # noqa: E731
                       [(c["slack"]["min"], c["slack"]["max"]) for c in r["constraints"]])
    assert strip(runs[0]) == strip(runs[1]) == strip(runs[2])


# ---- special ends -------------------------------------------------------------------------------------------------
UNB = {"optimize": "profit", "opType": "max",
       "constraints": {"cap": {"max": 7.5}, "link": {"max": 3}},
       "variables": {"x": {"profit": 2, "cap": 2}, "y": {"link": 1}, "z": {"link": -1}},
       "ints": {"x": 1}}


def test_an_unbounded_end_agrees_with_highs():
    got = MO.variability(UNB, width=2)
    assert got["exact"]
    assert got["variables"]["z"]["max"] == math.inf and got["variables"]["y"]["max"] == math.inf
    _, c, _, _ = lp_data(UNB)
    m = Model().loadJson(UNB)
    z_index = [v.id for v in m.variables].index("z")
    st, _ = highs(UNB, np.eye(3)[z_index], 1, (c, got["optimum"] - 1e-9, False))
    assert st == 3
    same_ranges(got, UNB)


@pytest.mark.parametrize("name, max_nodes", [("Knapsack 1.json", 100), ("Sudoku4x4.json", 3)])
def test_the_node_limit_reports_witnessed_ends_and_bounds(name, max_nodes):
    jm = fixture(name)
    full = MO.variability(jm, gap=0.01, width=4)
    part = MO.variability(jm, gap=0.01, width=4, max_nodes=max_nodes)
    assert full["exact"] and not part["exact"]
    limited = 0
    for vid, e in part["variables"].items():
        f = full["variables"][vid]
        assert f["min"] - 1e-9 <= e["min"] and e["max"] <= f["max"] + 1e-9
        if "bound" in e:
            limited += 1
            assert e["exact"] is False
            if "min" in e["bound"]:
                assert e["bound"]["min"] <= f["min"] + 1e-9
            if "max" in e["bound"]:
                assert e["bound"]["max"] >= f["max"] - 1e-9
    assert limited > 0


# ---- front end ----------------------------------------------------------------------------------------------------
KNAP = {"optimize": "v", "opType": "max", "constraints": {"w": {"max": 5}},
        "variables": {"a": {"v": 3, "w": 2}, "b": {"v": 4, "w": 3}}, "ints": {"a": 1, "b": 1}}


@pytest.mark.parametrize("model, kw, match", [
    ({**KNAP, "ints": {}}, {}, r"integer or binary.*variability\(\)"),
    ({**KNAP, "constraints": {"w": {"max": 5, "weight": 2}}}, {}, "soft constraints"),
    ({**KNAP, "optimize": {"v": "max", "w": "min"}}, {}, "one objective"),
    ({**KNAP, "unrestricted": {"a": 1}}, {}, "unrestricted"),
    ({**KNAP, "external": {"solver": "lpsolve"}}, {}, "external"),
    (KNAP, {"gap": -0.1}, "gap= must be finite and >= 0"),
    (KNAP, {"absolute_gap": float("nan")}, "absolute_gap= must be finite"),
    (KNAP, {"max_nodes": 0}, "max_nodes= must be >= 1"),
    (KNAP, {"width": 0}, "width= must be >= 1"),
    (KNAP, {"width": 1.5}, "width= takes an integer"),
    (KNAP, {"variables": "a"}, "variables= takes a list"),
    (KNAP, {"variables": ["nope"]}, "no variable named"),
    (KNAP, {"constraints": ["nope"]}, "no constraint named"),
    ([], {}, "requires a model"),
    ("model", {}, "takes a JSON model"),
])
def test_variability_refusals(model, kw, match):
    import jslpsolver_b200 as J
    with pytest.raises(ValueError, match=match):
        J.Variability(model, **kw)


INFEASIBLE = {"optimize": "v", "opType": "max", "constraints": {"odd": {"equal": 3}},
              "variables": {"a": {"v": 1, "odd": 2}, "b": {"v": 1, "odd": 2}}, "ints": {"a": 1, "b": 1}}
UNBOUNDED = {"optimize": "v", "opType": "max", "constraints": {"c": {"min": 1}},
             "variables": {"a": {"v": 1, "c": 1}}, "ints": {"a": 1}}


@pytest.mark.parametrize("model, kw, match", [
    (INFEASIBLE, {}, r"no integer plan.*Conflict\(\)"),
    (UNBOUNDED, {}, "unbounded"),
    (fixture("Knapsack 1.json"), {"max_nodes": 2}, "max_nodes"),
])
def test_restatement_refusals(model, kw, match):
    with pytest.raises(ValueError, match=match):
        MO.variability(model, **kw)


# ---- C ABI --------------------------------------------------------------------------------------------------------
def test_target_batch_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    C, P = _lib.C, _lib.C.c_void_p
    want = ["jslp_tab *", "const jslp_scenario_edit *", "const int32_t *", "const jslp_cut *", "const int32_t *",
            "int", "int", "int", "int32_t *", "double *", "int32_t *", "int32_t *", "double *", "int32_t *",
            "double *", "int32_t *"]
    assert _types("jslp_target_batch") == want
    (_, res, got), = [s for s in _lib.SYMBOLS if s[0] == "jslp_target_batch"]
    assert res is C.c_int and got == [P] * 5 + [C.c_int] * 3 + [P] * 8

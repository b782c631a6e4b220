"""Lexicographic objectives of a MIP (DESIGN.md section 2q) without a GPU: the restatement of
tests/lexicographic_mip_oracle.py against SciPy's HiGHS `milp` level by level (each level a MIP of its own under the
rows, the integrality and every earlier objective within its allowance) and against brute force; the final plan; level
1 against the oracle's Solve(); a huge allowance, monotone gaps and width invariance; every kind and stop; and
LexicographicMIP()'s refusals."""
from __future__ import annotations

import itertools
import re

import numpy as np
import pytest

import lexicographic_mip_oracle as LMO
from helpers import strip_timeouts
from jslpsolver_b200 import problems
from jslpsolver_b200.frontier import _coef
from jslpsolver_b200.model import object_keys
from test_mip_variability_cpu import SMALL, lp_data
from test_pool_cpu import fixture

REL = 1e-6


@pytest.fixture(scope="module", autouse=True)
def _oracle_lib():
    from oracle import ref_model
    ref_model.build_oracle()


def with_extra(jm: dict, senses, seed: int, lo: int = 0, hi: int = 20) -> dict:
    """jm with seeded extra objectives extra1.. of the given senses after its own objective (if it has one)."""
    rng = np.random.default_rng(seed)
    jm = strip_timeouts(jm)
    jm = dict(jm, variables={k: dict(v) for k, v in jm["variables"].items()})
    names = [f"extra{k + 1}" for k in range(len(senses))]
    for v in jm["variables"].values():
        for n in names:
            v[n] = float(rng.integers(lo, hi + 1))
    own = {jm["optimize"]: "max" if jm.get("opType") == "max" else "min"} if jm.get("optimize") else {}
    return dict(jm, optimize={**own, **dict(zip(names, senses))})


class Milp:
    """The JSON model's rows and integrality as loadJson reads them, one objective vector per `optimize` key."""

    def __init__(self, jm: dict):
        keys = object_keys(jm["optimize"])
        self.keys, self.sense = keys, {k: jm["optimize"][k] for k in keys}
        m, _, rows, self.integrality = lp_data(dict(jm, optimize=keys[0], opType=self.sense[keys[0]]))
        self.ids = [v.id for v in m.variables]
        self.rows = rows
        self.A = np.array([a for _, a in rows])
        self.lo = np.array([-np.inf if con.isUpperBound else con.rhs for con, _ in rows])
        self.hi = np.array([con.rhs if con.isUpperBound else np.inf for con, _ in rows])
        self.c = {k: np.array([_coef(jm, vid, k) for vid in self.ids]) for k in keys}

    def level(self, k: int, opt, allow):
        """(status, optimum) of objective k over the integer plans within allow[j] of opt[j] on every objective j < k;
        status 0 optimal, 2 infeasible, 3 unbounded (scipy.optimize.milp)."""
        from scipy.optimize import Bounds, LinearConstraint, milp
        cons = [LinearConstraint(self.A, self.lo, self.hi)]
        for j in range(k):
            key = self.keys[j]
            slack = allow[j] + 1e-9 * max(1.0, abs(opt[j]))
            if self.sense[key] == "max":
                cons.append(LinearConstraint(self.c[key][None, :], opt[j] - slack, np.inf))
            else:
                cons.append(LinearConstraint(self.c[key][None, :], -np.inf, opt[j] + slack))
        s = 1.0 if self.sense[self.keys[k]] == "max" else -1.0
        for presolve in (True, False):  # HiGHS's presolve reports "infeasible or unbounded" (4)
            res = milp(-s * self.c[self.keys[k]], constraints=cons, integrality=self.integrality,
                       bounds=Bounds(0, np.inf), options={"mip_rel_gap": 0, "presolve": presolve})
            if res.status != 4:
                break
        return res.status, (None if res.status != 0 else -s * res.fun)

    def check_plan(self, values: dict, opt, allow, P: float):
        x = np.array([values[v] for v in self.ids])
        scale = max(1.0, float(np.abs(x).max(initial=0.0)))
        assert np.all(np.abs(x[self.integrality == 1] - np.round(x[self.integrality == 1])) <= P * scale)
        assert np.all(x >= -P * scale)
        act = self.A @ x
        tol = 1e-7 * np.maximum(1.0, np.abs(np.where(np.isfinite(self.hi), self.hi, self.lo))) * scale
        assert np.all(act <= self.hi + tol) and np.all(act >= self.lo - tol)
        for j, (z, t) in enumerate(zip(opt, allow)):
            key = self.keys[j]
            loss = z - self.c[key] @ x if self.sense[key] == "max" else self.c[key] @ x - z
            assert loss <= t + 1e-7 * max(1.0, abs(z)) * scale, (key, loss, t)


def close(a: float, b: float) -> bool:
    return abs(a - b) <= REL * max(1.0, abs(a), abs(b))


def check_chain(jm: dict, **kw):
    """The restatement of jm against HiGHS level by level, and its final plan; returns (result, details)."""
    res, det = LMO.chain(jm, **kw)
    h = Milp(jm)
    if not res["feasible"]:
        assert h.level(0, [], [])[0] == 2
        return res, det
    opt, allow = [], []
    for k, lv in enumerate(res["levels"]):
        if lv["optimum"] is None:
            assert res["stop"] in ("unbounded", "cycled") and k == len(res["levels"]) - 1
            if res["stop"] == "unbounded":
                assert h.level(k, opt, allow)[0] == 3, (k, "HiGHS finds a bounded level")
            break
        if lv["exact"]:
            st, want = h.level(k, opt, allow)
            assert st == 0 and close(lv["optimum"], want), (k, lv["objective"], lv["optimum"], want)
        opt.append(lv["optimum"])
        allow.append(lv["allowance"] if lv["allowance"] is not None else 0.0)
    if res["values"] is not None:
        h.check_plan(res["values"], opt[:len(opt) - (res["stop"] == "reached")], allow, 1e-6)
    return res, det


# ---- against HiGHS ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SMALL)
@pytest.mark.parametrize("gap", [0.0, 0.05])
def test_bundle_chains_match_highs(name, gap):
    res, _ = check_chain(with_extra(fixture(name), ["min", "max"], seed=3), gap=gap, width=4)
    assert res["stop"] == "reached" and all(lv["exact"] for lv in res["levels"])


def generated():
    return [problems.random_mip_model(8, 5, seed=5, integer_fraction=0.6),
            problems.random_mip_model(10, 6, seed=11, integer_fraction=0.6),
            problems.knapsack_mip_model(12, 3, seed=4), problems.half_tie_mip_model(12, group=4)]


@pytest.mark.parametrize("jm", generated(), ids=lambda m: m["name"])
@pytest.mark.parametrize("senses", [["min"], ["max", "min"], ["min", "max", "min"]], ids=len)
@pytest.mark.parametrize("kw", [{"gap": 0.0}, {"gap": 0.05}, {"absolute_gap": {"extra1": 4.0}}], ids=str)
def test_generated_chains_match_highs(jm, senses, kw):
    res, _ = check_chain(with_extra(jm, senses, seed=7, lo=-5, hi=20), width=8, **kw)
    assert len(res["levels"]) == len(senses) + 1 or res["stop"] != "reached"


# ---- against brute force ---------------------------------------------------------------------------------------------
def pure_integer_models(n: int) -> list:
    """Seeded all-integer models (4 variables, 3 packing rows) with three objectives of mixed senses."""
    out = []
    for seed in range(n):
        rng = np.random.default_rng(100 + seed)
        names = [f"x{j}" for j in range(4)]
        A = rng.integers(1, 7, size=(3, 4))
        b = rng.integers(8, 21, size=3)
        variables = {v: {f"r{i}": int(A[i, j]) for i in range(3)} for j, v in enumerate(names)}
        keys = ["a", "b", "c"]
        for v in variables.values():
            for k in keys:
                v[k] = int(rng.integers(-4, 7))
        senses = ["max", "min", "max"] if seed % 2 == 0 else ["min", "max", "max"]
        out.append({"name": f"pure{seed}", "optimize": dict(zip(keys, senses)), "variables": variables,
                    "constraints": {f"r{i}": {"max": int(b[i])} for i in range(3)}, "ints": {v: 1 for v in names}})
    return out


def brute(jm: dict, gap: float, absolute_gap: float) -> list:
    """The lexicographic optima over every integer point, with the allowances of section 2q."""
    names = list(jm["variables"])
    rows = [(np.array([jm["variables"][v].get(r, 0) for v in names]), spec["max"])
            for r, spec in jm["constraints"].items()]
    box = [min(int(spec // a[j]) for a, spec in rows if a[j] > 0) for j in range(len(names))]
    pts = [np.array(p) for p in itertools.product(*[range(u + 1) for u in box])
           if all(a @ np.array(p) <= spec for a, spec in rows)]
    opts = []
    for key, sense in jm["optimize"].items():
        c = np.array([jm["variables"][v].get(key, 0) for v in names])
        vals = [float(c @ p) for p in pts]
        z = max(vals) if sense == "max" else min(vals)
        opts.append(z)
        t = max(absolute_gap, gap * abs(z))
        pts = [p for p, f in zip(pts, vals) if (z - f if sense == "max" else f - z) <= t + 1e-9]
    return opts


@pytest.mark.parametrize("jm", pure_integer_models(6), ids=lambda m: m["name"])
@pytest.mark.parametrize("gap, absolute_gap", [(0.0, 0.0), (0.1, 0.0), (0.0, 3.0)])
def test_restatement_matches_brute_force(jm, gap, absolute_gap):
    res, _ = LMO.chain(jm, gap=gap, absolute_gap=absolute_gap, width=2)
    assert res["stop"] == "reached"
    want = brute(jm, gap, absolute_gap)
    assert [lv["optimum"] for lv in res["levels"]] == pytest.approx(want, abs=1e-7)


# ---- properties of the answer ----------------------------------------------------------------------------------------
def test_level_one_is_solve_of_the_first_objective():
    from oracle import ref_model
    for jm in [with_extra(fixture(n), ["max"], seed=1) for n in SMALL[:6]] + \
              [with_extra(m, ["min"], seed=2) for m in generated()]:
        res, _ = LMO.chain(jm, width=4)
        key = object_keys(jm["optimize"])[0]
        single = dict(jm, optimize=key, opType=jm["optimize"][key], options={"presolve": False})
        sol = ref_model.solve_full(single)
        if res["stop"] == "unbounded":
            assert not sol.bounded and len(res["levels"]) == 1, jm["name"]
            continue
        assert abs(res["levels"][0]["optimum"] - sol.evaluation) <= 1e-8 * max(1.0, abs(sol.evaluation)), jm["name"]


def test_a_huge_allowance_makes_level_two_the_second_objective_alone():
    for jm in [with_extra(fixture("Knapsack 1.json"), ["min"], seed=5), with_extra(generated()[1], ["max"], seed=6)]:
        res, _ = LMO.chain(jm, absolute_gap=1e9, width=8)
        h = Milp(jm)
        alone = Milp(dict(jm, optimize={h.keys[1]: h.sense[h.keys[1]]}))
        assert close(res["levels"][1]["optimum"], alone.level(0, [], [])[1])


def test_later_optima_are_monotone_in_the_gap():
    jm = with_extra(fixture("Knapsack 1.json"), ["min", "max"], seed=3)
    last = None
    for gap in (0.0, 0.01, 0.05, 0.2):
        res, _ = LMO.chain(jm, gap=gap, width=8)
        opt = res["levels"][1]["optimum"]
        if last is not None:
            assert opt <= last + 1e-9  # extra1 is minimised: a wider allowance can only lower it
        last = opt


@pytest.mark.parametrize("name", ["Knapsack 1.json", "Integer Sports Complex Problem.json", "Sudoku4x4.json"])
def test_width_changes_no_optimum(name):
    jm = with_extra(fixture(name), ["min", "max"], seed=4)
    runs = [LMO.chain(jm, gap=0.02, **kw)[0] for kw in ({"width": 1}, {"wave": 256}, {"width": 64})]
    for r in runs[1:]:
        assert [lv["optimum"] for lv in r["levels"]] == [lv["optimum"] for lv in runs[0]["levels"]]
        assert r["values"] == runs[0]["values"]


# ---- kinds and stops -------------------------------------------------------------------------------------------------
POINT = {"name": "point", "optimize": {"v": "max", "w": "min", "u": "max"},
         "constraints": {"a": {"max": 3}, "b": {"max": 2}},
         "variables": {"x": {"v": 1, "w": 1, "u": 2, "a": 1}, "y": {"v": 2, "w": 3, "u": 1, "b": 1}},
         "ints": {"x": 1, "y": 1}}
INFEASIBLE = {"name": "odd", "optimize": {"v": "max", "w": "min"}, "constraints": {"odd": {"equal": 3}},
              "variables": {"a": {"v": 1, "w": 1, "odd": 2}, "b": {"v": 1, "w": 2, "odd": 2}}, "ints": {"a": 1, "b": 1}}
UNBOUNDED_1 = {"name": "unb1", "optimize": {"v": "max", "w": "min"}, "constraints": {"c": {"min": 1}},
               "variables": {"a": {"v": 1, "w": 1, "c": 1}}, "ints": {"a": 1}}
UNBOUNDED_2 = {"name": "unb2", "optimize": {"profit": "max", "y": "max"},
               "constraints": {"cap": {"max": 7.5}, "link": {"max": 3}},
               "variables": {"x": {"profit": 2, "cap": 2}, "y": {"link": 1, "y": 1}, "z": {"link": -1}},
               "ints": {"x": 1}}


def zero_first(jm: dict) -> dict:
    """jm with an all-zero objective in front of its own: level 1 ends at its root, level 2 is jm's own search."""
    return dict(strip_timeouts(jm), optimize={"nothing": "min", jm["optimize"]: jm.get("opType", "min")})


def test_face_and_bound_levels():
    """An all-zero first objective: its MIP optimum is its LP optimum, so at gap 0 level 2 runs on the optimal face
    (every column, since every reduced cost is 0); a gap makes it a bound tableau."""
    jm = dict(with_extra(fixture("Sudoku4x4.json"), ["min"], seed=2), optimize={"nothing": "min", "extra1": "min"})
    res, det = check_chain(jm, width=8)
    assert [lv["kind"] for lv in res["levels"]] == ["initial", "face"] and det[0]["delta"] == 0.0
    assert res["levels"][1]["width"] == res["levels"][0]["width"]
    res, _ = check_chain(with_extra(fixture("Knapsack 1.json"), ["min"], seed=2), gap=0.01, width=8)
    assert res["levels"][1]["kind"] == "bound"


def test_a_single_point_face_ends_the_search():
    res, det = check_chain(POINT, width=2)
    assert [lv["kind"] for lv in res["levels"]] == ["initial", None, None]
    assert res["values"] == {"x": 3.0, "y": 2.0}
    assert [lv["optimum"] for lv in res["levels"]] == [7.0, 9.0, 8.0]
    assert res["levels"][1]["nodes"] == 0 and det[1]["level"] is None


def test_no_integer_plan():
    res, _ = check_chain(INFEASIBLE, width=2)
    assert not res["feasible"] and res["stop"] is None and len(res["levels"]) == 1 and res["values"] is None


def test_unbounded_at_level_one_and_at_level_two():
    res, _ = check_chain(UNBOUNDED_1, width=2)
    assert (res["stop"], res["bounded"], res["values"], len(res["levels"])) == ("unbounded", False, None, 1)
    res, _ = check_chain(UNBOUNDED_2, width=2)
    assert (res["stop"], res["bounded"], len(res["levels"])) == ("unbounded", False, 2)
    assert res["levels"][0]["optimum"] == 6.0 and res["values"]["x"] == 3.0


def test_the_node_limit():
    jm = zero_first(fixture("Knapsack 1.json"))
    full, _ = check_chain(jm, width=4)
    part, _ = LMO.chain(jm, width=4, max_nodes=5)
    assert full["stop"] == "reached" and part["stop"] == "limit"
    lv = part["levels"][1]
    assert lv["exact"] is False and lv["bound"] >= full["levels"][1]["optimum"] - 1e-9  # extra is maximised
    assert lv["optimum"] <= full["levels"][1]["optimum"] + 1e-9
    assert part["values"] is not None
    with pytest.raises(ValueError, match="raise max_nodes"):
        LMO.chain(fixture_knapsack_two(), width=4, max_nodes=2)


KNAP20 = problems.knapsack_mip_model(20, 3, seed=4)  # MIP optimum 381; a search of 5 nodes evaluates it at width 4


@pytest.mark.parametrize("max_nodes", [5, 10, 20])
def test_a_limit_keeps_the_best_integral_node_it_evaluated(max_nodes):
    """At a later level the limit reports the best integral node the level evaluated, not the level before's plan."""
    res, _ = LMO.chain(zero_first(KNAP20), width=4, max_nodes=max_nodes)
    assert res["stop"] == "limit" and res["levels"][0]["optimum"] == 0.0
    lv = res["levels"][1]
    assert lv["exact"] is False and lv["optimum"] == 381.0 and lv["bound"] >= 381.0
    h = Milp(zero_first(KNAP20))
    assert h.level(1, [0.0], [0.0]) == (0, pytest.approx(381.0))
    h.check_plan(res["values"], [0.0], [0.0], 1e-6)
    assert res["objectives"][KNAP20["optimize"]] == pytest.approx(381.0)


@pytest.mark.parametrize("max_nodes", [5, 20])
def test_a_limit_at_level_one_after_an_integral_node_is_a_stop(max_nodes):
    """Level 1 raises only when no integral node was evaluated; with one, the limit is a stop with that plan."""
    jm = dict(KNAP20, optimize={KNAP20["optimize"]: "max", "nothing": "min"})
    res, _ = LMO.chain(jm, width=4, max_nodes=max_nodes)
    assert res["stop"] == "limit" and len(res["levels"]) == 1
    lv = res["levels"][0]
    assert lv["exact"] is False and lv["optimum"] == 381.0 and lv["bound"] >= 381.0
    Milp(jm).check_plan(res["values"], [], [], 1e-6)


def test_a_constant_later_objective_cycles():
    """An all-zero objective after a MIP: every node LP of its level has a zero cost row on a degenerate optimum, the
    simplex's cycle check fires, and the call reports stop "cycled" with level 1's plan (DESIGN section 2q)."""
    jm = dict(KNAP20, optimize={KNAP20["optimize"]: "max", "nothing": "min"})
    res, _ = LMO.chain(jm, width=4)
    assert res["stop"] == "cycled" and res["levels"][0]["optimum"] == 381.0 and res["values"] is not None


def fixture_knapsack_two() -> dict:
    return with_extra(fixture("Knapsack 1.json"), ["min"], seed=1)


# ---- refusals --------------------------------------------------------------------------------------------------------
KNAP = {"optimize": {"v": "max", "w": "min"}, "constraints": {"w": {"max": 5}},
        "variables": {"a": {"v": 3, "w": 2}, "b": {"v": 4, "w": 3}}, "ints": {"a": 1, "b": 1}}


@pytest.mark.parametrize("model, kw, match", [
    ({**KNAP, "ints": {}}, {}, r"integer or binary.*Lexicographic\(\)"),
    ({**KNAP, "optimize": {"v": "max"}}, {}, "at least two"),
    ({**KNAP, "optimize": "v"}, {}, "at least two"),
    ({**KNAP, "constraints": {"w": {"max": 5, "weight": 2}}}, {}, "soft constraints"),
    ({**KNAP, "constraints": {"w": {"max": 5, "priority": "strong"}}}, {}, "soft constraints"),
    ({**KNAP, "unrestricted": {"a": 1}}, {}, "unrestricted"),
    (KNAP, {"gap": -0.1}, "gap= must be finite and >= 0"),
    (KNAP, {"gap": {"nope": 0.1}}, "names 'nope'"),
    (KNAP, {"absolute_gap": float("nan")}, "absolute_gap= must be finite"),
    (KNAP, {"absolute_gap": True}, "absolute_gap= takes a number"),
    (KNAP, {"max_nodes": 0}, "max_nodes= must be >= 1"),
    (KNAP, {"max_nodes": 2.0}, "max_nodes= takes an integer"),
    (KNAP, {"width": 0}, "width= must be >= 1"),
    (KNAP, {"width": 1.5}, "width= takes an integer"),
    ("model", {}, "takes a JSON model"),
])
def test_refusals(model, kw, match):
    import jslpsolver_b200 as J
    with pytest.raises(ValueError, match=r"LexicographicMIP\(\).*" + match):
        J.LexicographicMIP(model, **kw)


def test_other_refusals_and_the_exports():
    import jslpsolver_b200 as J
    with pytest.raises(ValueError, match=re.escape("requires a model")):
        J.LexicographicMIP({})
    with pytest.raises(NotImplementedError):
        J.LexicographicMIP({**KNAP, "external": {"solver": "lpsolve"}})
    assert J.Solver.LexicographicMIP is not None and "LexicographicMIP" in J.__all__
    # Lexicographic() keeps refusing MIPs, with its own message
    with pytest.raises(ValueError, match=r"Lexicographic\(\) is defined for continuous LPs only"):
        J.Lexicographic(KNAP)

"""Repair of an infeasible MIP (DESIGN.md section 2r) without a GPU: the restatement of tests/repair_mip_oracle.py
against SciPy's HiGHS `milp` on the elastic MIP (the model's tableau rows with a violation e_j >= 0 on each relaxable
row, integrality, minimise sum w e; stage 2 the model's objective with sum w e <= V* + t added) and against brute
force on tiny binary models; the properties of the answer (an integral plan that meets its repaired rows, Solve() of
the repaired model, V* against Repair() of the LP relaxation, a feasible MIP, stage 2 monotone in t); every stop; and
RepairMIP()'s refusals, with Repair()'s refusal of MIPs unchanged."""
from __future__ import annotations

import itertools
import math
import re

import numpy as np
import pytest

import pool_oracle as PO
import repair_mip_oracle as RMO
import repair_oracle as RO
from helpers import strip_timeouts
from jslpsolver_b200 import problems
from jslpsolver_b200.frontier import _coef
from test_conflict_cpu import EXAMPLE, infeasible_berlin_with_ints, random_infeasible_mips
from test_gpu_pool import beale_mip

REL = 1e-6


@pytest.fixture(scope="module", autouse=True)
def _oracle_lib():
    from oracle import ref_model
    ref_model.build_oracle()


def with_ints(jm: dict) -> dict:
    return dict(jm, ints={v: 1 for v in jm["variables"]})


def unbounded_stage_two() -> dict:
    """`2x = 3` with x integer, and y free to grow without any row: stage 2 runs away along y."""
    return {"optimize": "z", "opType": "max", "constraints": {"pair": {"equal": 3}},
            "variables": {"x": {"pair": 2}, "y": {"z": 1}}, "ints": {"x": 1}}


KNAP20 = problems.knapsack_mip_model(20, 3, seed=4)  # feasible: V* = 0 at the root, stage 2 its MIP optimum 381
PACK = with_ints(problems.infeasible_packing_model(8, 8, 2, seed=3))


def infeasible_families() -> dict:
    return {"example": EXAMPLE, "berlin": infeasible_berlin_with_ints(),
            "planted1": problems.planted_integer_conflict_model(6, 5, 2, seed=1),
            "planted2": problems.planted_integer_conflict_model(12, 10, 3, seed=2),
            **{f"random{i}": m for i, m in enumerate(random_infeasible_mips(3))},
            "packing3": PACK, "packing5": with_ints(problems.infeasible_packing_model(10, 8, 3, seed=5))}


FAMILIES = infeasible_families()


# ---- HiGHS ----------------------------------------------------------------------------------------------------------
class Elastic:
    """The elastic MIP of a JSON model over its initial tableau (every tableau row r reads M[r,1:] x <= M[r,0]): the
    relaxable row r_j gets -e_j, integrality on the integer labels' columns, and the model's objective by column."""

    def __init__(self, jm: dict, rows, weights):
        self.p = p = PO.Problem(strip_timeouts(jm))
        M = p.M
        H, W = M.shape
        k = len(rows)
        self.A = np.zeros((H - 1, W - 1 + k))
        self.A[:, :W - 1] = M[1:, 1:]
        for j, r in enumerate(rows):
            self.A[r - 1, W - 1 + j] = -1.0
        self.b = M[1:, 0].copy()
        self.w = np.concatenate([np.zeros(W - 1), np.asarray(weights, dtype=float)])
        self.integrality = np.zeros(W - 1 + k)
        for lab in p.ints:
            self.integrality[p.col_of[lab] - 1] = 1
        self.cols = [p.col_of[v.index] - 1 for v in p.m.variables]
        key = jm.get("optimize") if isinstance(jm.get("optimize"), str) else None
        self.c = np.zeros(W - 1 + k)
        for v, c in zip(p.m.variables, self.cols):
            self.c[c] = _coef(jm, v.id, key) if key is not None else 0.0
        self.sense = "max" if jm.get("opType") == "max" else "min"

    def solve(self, cap=None):
        """(status, optimum): stage 1 (cap None), or the objective subject to w.e <= cap; status 0 optimal,
        2 infeasible, 3 unbounded (scipy.optimize.milp)."""
        from scipy.optimize import Bounds, LinearConstraint, milp
        cons = [LinearConstraint(self.A, -np.inf, self.b)]
        if cap is None:
            c, s = self.w, 1.0
        else:
            cons.append(LinearConstraint(self.w[None, :], -np.inf, cap))
            s = -1.0 if self.sense == "max" else 1.0
            c = s * self.c
        for presolve in (True, False):  # HiGHS's presolve reports "infeasible or unbounded" (4)
            res = milp(c, constraints=cons, integrality=self.integrality, bounds=Bounds(0, np.inf),
                       options={"mip_rel_gap": 0, "presolve": presolve})
            if res.status != 4:
                break
        return res.status, (None if res.status != 0 else s * res.fun)

    def check_plan(self, res: dict):
        """The plan is integral, non-negative and meets every row at its repaired right-hand side."""
        p = self.p
        vals = np.array([res["values"][v.id] for v in p.m.variables])
        scale = max(1.0, float(np.abs(vals).max(initial=0.0)))
        ints = [i for i, v in enumerate(p.m.variables) if v.index in set(p.ints)]
        assert np.all(np.abs(vals[ints] - np.round(vals[ints])) <= 1e-7 * scale)
        assert np.all(vals >= -1e-9 * scale)
        x = np.zeros(p.M.shape[1] - 1)
        x[self.cols] = vals
        row_of = {(name if name is not None else con.index, "max" if con.isUpperBound else "min"): r
                  for r, (con, name) in enumerate(zip(p.m.constraints, names_of(p)))}
        relaxed = np.zeros(len(self.b))
        for c in res["constraints"]:
            relaxed[row_of[(c["name"], c["type"])]] = c["violation"]
        act = p.M[1:, 1:] @ x
        tol = 1e-7 * np.maximum(1.0, np.abs(self.b)) * scale
        assert np.all(act <= self.b + relaxed + tol), (act - self.b - relaxed).max()


def names_of(p) -> list:
    from oracle.sensitivity import json_row_names
    names = json_row_names(p.jm)
    return names + [None] * (len(p.m.constraints) - len(names))


def close(a: float, b: float) -> bool:
    return abs(a - b) <= REL * max(1.0, abs(a), abs(b))


def check(jm: dict, weights=None, **kw):
    """The restatement of jm against HiGHS, stage by stage, and its plan; returns (result, details)."""
    res, det = RMO.repair_mip(jm, weights, **kw)
    h = Elastic(jm, det["rows"], det["weights"])
    st, vstar = h.solve()
    if not res["feasible"]:
        assert st == 2 and res["stop"] == "infeasible" and res["values"] is None
        return res, det
    s1 = res["stages"][0]
    if res["stop"] == "cycled" and res["values"] is None:
        return res, det
    assert st == 0
    if s1["exact"]:
        assert close(s1["optimum"], vstar), (s1["optimum"], vstar)
    else:
        assert s1["bound"] <= vstar + 1e-7 and s1["optimum"] >= vstar - 1e-7
    if len(res["stages"]) > 1:
        s2 = res["stages"][1]
        st2, z = h.solve(s1["optimum"] + s2["allowance"] + 1e-9 * max(1.0, s1["optimum"]))
        if res["stop"] == "unbounded":
            assert st2 == 3
        elif s2["exact"] and s2["optimum"] is not None:
            assert st2 == 0 and close(s2["optimum"], z), (s2["optimum"], z)
    h.check_plan(res)
    if res["stop"] == "reached" and len(res["stages"]) > 1:
        assert res["violation"] <= s1["optimum"] + res["stages"][1]["allowance"] + 1e-7 * max(1.0, s1["optimum"])
        assert close(res["result"], res["stages"][1]["optimum"])
    return res, det


# ---- against HiGHS --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(FAMILIES))
@pytest.mark.parametrize("kw", [{"width": 4}, {"gap": 0.05, "width": 16}, {"absolute_gap": 2.0, "width": 1},
                                {"objective": False, "width": 4}], ids=str)
def test_infeasible_families_match_highs(name, kw):
    res, _ = check(FAMILIES[name], **kw)
    assert res["feasible"] and res["stages"][0]["optimum"] > 0.0
    assert len(res["stages"]) == (1 if kw.get("objective") is False else 2) or res["stop"] != "reached"


def test_random_weight_subsets_match_highs():
    rng = np.random.default_rng(5)
    for name in ("planted2", "packing3", "random1"):
        jm = FAMILIES[name]
        names = list(jm["constraints"])
        for _ in range(2):
            pick = [n for n in names if rng.random() < 0.7] or names[:1]
            check(jm, {n: float(rng.uniform(0.5, 5.0)) for n in pick}, width=8)
    # only `cap` may move: the parity rows conflict with integrality on their own
    res, _ = check(EXAMPLE, {"cap": 1.0}, width=4)
    assert (res["feasible"], res["stop"], res["violation"], res["constraints"]) == (False, "infeasible", None, [])
    # planted: only one side of the parity row may move, with a weight
    res, _ = check(FAMILIES["planted1"], {"parity": {"max": 3.0}}, width=4)
    assert res["violation"] == 3.0 and [c["type"] for c in res["constraints"]] == ["max"]


# ---- against brute force --------------------------------------------------------------------------------------------
def tiny_binary_models(n: int) -> list:
    """Seeded binary models (4 items, 2 rows) whose rows no 0/1 point meets: a `min` cover row and an `equal` row."""
    out = []
    for seed in range(200):
        rng = np.random.default_rng(300 + seed)
        a, b = rng.integers(1, 6, size=4), rng.integers(1, 6, size=4)
        need, eq = int(rng.integers(5, 14)), int(rng.integers(2, 12))
        pts = list(itertools.product((0, 1), repeat=4))
        if any(np.dot(a, x) >= need and np.dot(b, x) == eq for x in pts):
            continue
        out.append({"name": f"tiny{seed}", "optimize": "v", "opType": "max" if seed % 2 else "min",
                    "constraints": {"cover": {"min": need}, "fit": {"equal": eq}},
                    "variables": {f"x{j}": {"v": int(rng.integers(-3, 8)), "cover": int(a[j]), "fit": int(b[j])}
                                  for j in range(4)},
                    "binaries": {f"x{j}": 1 for j in range(4)}})
        if len(out) == n:
            return out
    raise AssertionError("too few tiny infeasible binary models")


@pytest.mark.parametrize("jm", tiny_binary_models(6), ids=lambda m: m["name"])
@pytest.mark.parametrize("weights", [{"cover": 1.0, "fit": 1.0}, {"cover": 3.0, "fit": {"min": 1.0, "max": 0.5}}],
                         ids=["unit", "weighted"])
@pytest.mark.parametrize("gap", [0.0, 0.5])
def test_restatement_matches_brute_force(jm, weights, gap):
    """The binaries' own `x <= 1` rows are not named, so they stay hard and every plan is a 0/1 point."""
    res, _ = RMO.repair_mip(jm, weights, gap=gap, width=2)
    names = list(jm["variables"])
    wc = weights["cover"]
    wf = weights["fit"] if isinstance(weights["fit"], dict) else {"min": weights["fit"], "max": weights["fit"]}
    best = []
    for x in itertools.product((0, 1), repeat=4):
        cover = sum(jm["variables"][v]["cover"] * xi for v, xi in zip(names, x))
        fit = sum(jm["variables"][v]["fit"] * xi for v, xi in zip(names, x))
        eq = jm["constraints"]["fit"]["equal"]
        viol = wc * max(0, jm["constraints"]["cover"]["min"] - cover) + wf["min"] * max(0, eq - fit) + \
            wf["max"] * max(0, fit - eq)
        best.append((viol, sum(jm["variables"][v]["v"] * xi for v, xi in zip(names, x))))
    vstar = min(v for v, _ in best)
    t = gap * vstar
    allowed = [z for v, z in best if v <= vstar + t + 1e-9]
    want = max(allowed) if jm["opType"] == "max" else min(allowed)
    assert res["stop"] == "reached"
    assert res["stages"][0]["optimum"] == pytest.approx(vstar, abs=1e-9)
    assert res["result"] == pytest.approx(want, abs=1e-9) and res["stages"][1]["optimum"] == pytest.approx(want)


# ---- properties of the answer ---------------------------------------------------------------------------------------
def repaired_model(jm: dict, res: dict) -> dict:
    """jm with every violated row's right-hand side moved to its repairedRhs (loosened by 1e-9 relative) and
    presolve off."""
    cons = {k: dict(v) for k, v in jm["constraints"].items()}
    for c in res["constraints"]:
        spec = cons[c["name"]]
        if spec.get("equal") is not None:  # an equality relaxed on one side keeps the other
            lo = hi = spec.pop("equal")
            spec.update(min=lo, max=hi)
        r = c["repairedRhs"]
        spec[c["type"]] = r + (1e-9 if c["type"] == "max" else -1e-9) * max(1.0, abs(r))
    return dict(strip_timeouts(jm), constraints=cons, options={"presolve": False})


@pytest.mark.parametrize("name", list(FAMILIES))
def test_the_repaired_model_solves_to_the_result(name):
    from oracle import ref_model
    res, _ = RMO.repair_mip(FAMILIES[name], width=8)
    if res["stop"] != "reached":
        assert res["stop"] == "unbounded" and name == "random2"
        return
    sol = ref_model.Solve(repaired_model(FAMILIES[name], res))
    assert sol["feasible"]
    assert abs(sol["result"] - res["result"]) <= 1e-6 * max(1.0, abs(res["result"])), (sol["result"], res["result"])


@pytest.mark.parametrize("name", list(FAMILIES))
def test_vstar_is_at_least_the_repair_of_the_relaxation(name):
    jm = FAMILIES[name]
    res, _ = RMO.repair_mip(jm, width=8, objective=False)
    lp = {k: v for k, v in jm.items() if k not in ("ints", "binaries")}
    relaxed, _ = RO.repair(lp, objective=False)
    if relaxed["stop"] == "cycled":
        pytest.skip("the LP repair cycles")
    assert res["violation"] >= relaxed["violation"] - 1e-9
    if name in ("example", "planted1", "planted2"):  # the relaxation is feasible: only integrality breaks a row
        assert relaxed["violation"] == 0.0 and res["violation"] == 1.0


def test_the_example_of_the_readme():
    res, _ = RMO.repair_mip(EXAMPLE)
    assert (res["violation"], res["result"], res["values"]) == (1.0, 1.0, {"x": 1.0, "y": 0.0})
    assert res["constraints"] == [{"name": "pair", "type": "min", "rhs": 3, "weight": 1.0, "violation": 1.0,
                                   "repairedRhs": 2.0}]


@pytest.mark.parametrize("jm", [KNAP20, problems.knapsack_mip_model(12, 3, seed=4),
                                problems.random_mip_model(10, 6, seed=11, integer_fraction=0.6),
                                problems.half_tie_mip_model(12, group=4)], ids=lambda m: m["name"])
def test_a_feasible_mip_repairs_to_its_optimum(jm):
    from oracle import ref_model
    res, _ = check(jm, width=8)
    assert res["violation"] == 0.0 and res["constraints"] == [] and res["stop"] == "reached"
    want = ref_model.Solve(dict(strip_timeouts(jm), options={"presolve": False}))["result"]
    assert abs(res["result"] - want) <= 1e-6 * max(1.0, abs(want)), (res["result"], want)


@pytest.mark.parametrize("name", ["planted2", "packing3", "berlin"])
def test_stage_two_is_monotone_in_the_allowance(name):
    jm = FAMILIES[name]
    last = None
    for kw in ({}, {"gap": 0.01}, {"gap": 0.1}, {"absolute_gap": 5.0}, {"gap": 1.0}):
        res, _ = check(jm, width=8, **kw)
        s2 = res["stages"][1]
        if last is not None and s2["allowance"] >= last[0]:
            assert s2["optimum"] >= last[1] - 1e-9 * max(1.0, abs(last[1]))  # every family maximises
        last = (s2["allowance"], s2["optimum"])


@pytest.mark.parametrize("name", ["planted2", "packing5"])
def test_width_changes_no_optimum(name):
    runs = [RMO.repair_mip(FAMILIES[name], **kw)[0] for kw in ({"width": 1}, {"wave": 256}, {"width": 64})]
    for r in runs[1:]:
        assert [s["optimum"] for s in r["stages"]] == [s["optimum"] for s in runs[0]["stages"]]


# ---- stops ----------------------------------------------------------------------------------------------------------
def test_unbounded_stage_two_keeps_the_stage_one_plan():
    res, _ = check(unbounded_stage_two(), width=4)
    assert res["stop"] == "unbounded" and res["violation"] == 1.0 and res["stages"][1]["optimum"] is None
    assert res["values"]["x"] in (1.0, 2.0) and res["values"]["y"] == 0.0


def test_a_cycling_stage_two_keeps_the_stage_one_plan():
    """Beale's cycling LP, feasible: V* = 0 at the root and stage 2's root node cycles."""
    res, _ = check(beale_mip(), width=4)
    assert res["stop"] == "cycled" and res["violation"] == 0.0 and res["stages"][1]["optimum"] is None
    assert res["values"] is not None


@pytest.mark.parametrize("max_nodes", [3, 6, 9])
def test_a_limit_in_stage_one_keeps_the_best_integral_node(max_nodes):
    res, _ = check(PACK, width=4, max_nodes=max_nodes)
    s1 = res["stages"][0]
    assert res["stop"] == "limit" and len(res["stages"]) == 1 and s1["exact"] is False
    assert s1["bound"] <= 320.0 <= s1["optimum"] == res["violation"]


def test_a_limit_in_stage_one_before_any_integral_node_raises():
    with pytest.raises(ValueError, match=r"RepairMIP\(\): the search of stage 1 hit max_nodes=8 .*raise max_nodes"):
        RMO.repair_mip(with_ints(problems.infeasible_packing_model(20, 16, 4, seed=5)), width=4, max_nodes=8)


@pytest.mark.parametrize("max_nodes", [5, 20])
def test_a_limit_in_stage_two_keeps_the_best_integral_node(max_nodes):
    res, _ = check(KNAP20, width=4, max_nodes=max_nodes)
    s2 = res["stages"][1]
    assert res["stop"] == "limit" and res["stages"][0]["exact"] and s2["exact"] is False
    assert s2["optimum"] == 381.0 == res["result"] and s2["bound"] >= 381.0


# ---- refusals -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model, kw, match", [
    ({**EXAMPLE, "ints": {}}, {}, r"integer or binary.*Repair\(\)"),
    ({**EXAMPLE, "constraints": {"pair": {"equal": 3, "weight": 2}}}, {}, "soft constraints"),
    ({**EXAMPLE, "constraints": {"pair": {"equal": 3, "priority": "strong"}}}, {}, "soft constraints"),
    ({**EXAMPLE, "unrestricted": {"x": 1}}, {}, "unrestricted"),
    ({**EXAMPLE, "optimize": {"cost": "min", "x": "max"}}, {}, "one objective"),
    ({**EXAMPLE, "external": {"solver": "lpsolve"}}, {}, "external"),
    (EXAMPLE, {"gap": -0.1}, "gap= must be finite and >= 0"),
    (EXAMPLE, {"absolute_gap": math.nan}, "absolute_gap= must be finite"),
    (EXAMPLE, {"gap": True}, "gap= takes a number"),
    (EXAMPLE, {"max_nodes": 0}, "max_nodes= must be >= 1"),
    (EXAMPLE, {"max_nodes": 2.0}, "max_nodes= takes an integer"),
    (EXAMPLE, {"width": 0}, "width= must be >= 1"),
    (EXAMPLE, {"width": 1.5}, "width= takes an integer"),
    ("model", {}, "takes a JSON model"),
])
def test_refusals(model, kw, match):
    import jslpsolver_b200 as J
    with pytest.raises(ValueError, match=r"RepairMIP\(\).*" + match):
        J.RepairMIP(model, **kw)


def test_weight_errors_and_the_width_cap():
    from jslpsolver_b200.repair_mip import RepairMIP
    from test_repair_cpu import _StubSolver
    s = _StubSolver()
    for weights, match in (({"nope": 1.0}, "no constraint named 'nope'"), ({"cap": 0.0}, "must be finite and > 0"),
                           ({"cap": math.inf}, "finite and > 0"), ({"cap": True}, "must be a number"),
                           ({"cap": {}}, "needs a 'min'"), ({"cap": {"equal": 1}}, "side must be"),
                           ({"cap": {"min": 1.0}}, "only a 'max' bound"), ([1.0], "takes a dict")):
        with pytest.raises(ValueError, match=r"RepairMIP\(\).*" + re.escape(match)):
            RepairMIP(s, EXAMPLE, weights)
    wide = {"optimize": "z", "opType": "max", "constraints": {f"r{i}": {"max": 1} for i in range(25599)},
            "variables": {"x": {"z": 1, **{f"r{i}": 1 for i in range(25599)}}}, "ints": {"x": 1}}
    with pytest.raises(ValueError, match=r"RepairMIP\(\): the elastic tableau needs 25601 columns .*cap of 25600"):
        RepairMIP(s, wide)
    assert all(t.M is None for t in s.log), "a refused call uploaded a tableau"


def test_other_refusals_and_the_exports():
    import jslpsolver_b200 as J
    with pytest.raises(ValueError, match=re.escape("requires a model")):
        J.RepairMIP({})
    assert J.Solver.RepairMIP is not None and "RepairMIP" in J.__all__
    # Repair() keeps refusing MIPs, with its own message
    for jm in (EXAMPLE, dict(KNAP20)):
        with pytest.raises(ValueError, match=r"Repair\(\) is defined for continuous LPs only: the model has integer"):
            J.Repair(jm)

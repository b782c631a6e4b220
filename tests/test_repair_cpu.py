"""CPU checks of Repair() (DESIGN.md section 2k) over the restatement in repair_oracle.py.  Stage 1's V* equals SciPy
HiGHS's optimum of the elastic LP (the model's rows with `a.x - e <= b` / `a.x + e >= b` on the relaxable rows, e >= 0,
minimise sum w e) on the infeasible fixtures, planted_infeasible_model, infeasible_packing_model, mixed_lp_model,
random weights and weights= subsets; every plan meets its repaired rows and the model with the repaired right-hand
sides is feasible; every IIS of the deletion filter holds a violated row; stage 2 equals HiGHS's second stage and is
monotone in the allowance; a feasible model repairs to V* = 0 and Solve()'s result; stage 1 makes no phase-1 pivot
when every row may be relaxed; rule 1's row 0 is the fixed-order sum; the host driver over a stand-in tableau equals
the restatement; every refusal, weight error and the width cap; the C prototype."""
import math
import os
import re
import types

import numpy as np
import pytest

import repair_oracle as RO
from conftest import ROOT, load_bundle
from helpers import strip_timeouts

BUNDLE = load_bundle()
P = 1e-8
BERLIN = {"optimize": "capacity", "opType": "max",
          "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
          "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                        "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}
BROKEN = dict(BERLIN, constraints=dict(BERLIN["constraints"], brit={"min": 13}))


def _plain(jm):
    return not (jm.get("ints") or jm.get("binaries") or jm.get("unrestricted") or
                any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())) \
        and isinstance(jm.get("optimize"), str)


INFEASIBLE = [f for f in BUNDLE["fixtures"] if not f["expects"].get("feasible", True) and _plain(f["model"])]


def _rows(jm):
    """[(name, 'max' | 'min', a, b)] in tableau row order: `min` before `max`, an `equal` as min then max.  A
    constraint named like the objective has no terms: loadJson reads those coefficients as costs only."""
    names = list(jm["variables"])
    out = []
    for cname, spec in jm["constraints"].items():
        a = np.array([0.0 if cname == jm.get("optimize") else float(jm["variables"][v].get(cname, 0.0))
                      for v in names])
        if spec.get("equal") is not None:
            out += [(cname, "min", a, float(spec["equal"])), (cname, "max", a, float(spec["equal"]))]
        else:
            out += [(cname, s, a, float(spec[s])) for s in ("min", "max") if spec.get(s) is not None]
    return names, out


def highs_elastic(jm, rows, weights, second=None):
    """HiGHS on the elastic LP: V* (second=None), or with second = (V* + t, sense) the model's objective optimised
    subject to sum w e <= V* + t.  Returns the optimum, None when infeasible, +-inf when unbounded."""
    from scipy.optimize import linprog
    names, R = _rows(jm)
    n, k = len(names), len(rows)
    col = {r: j for j, r in enumerate(rows)}
    A, b = [], []
    for i, (_, kind, a, rhs) in enumerate(R, start=1):
        e = np.zeros(k)
        if i in col:
            e[col[i]] = -1.0
        if kind == "max":
            A.append(np.concatenate([a, e])); b.append(rhs)
        else:
            A.append(np.concatenate([-a, e])); b.append(-rhs)
    w = np.concatenate([np.zeros(n), np.asarray(weights, dtype=float)])
    if second is None:
        c = w
        s = 1.0
    else:
        cap, sense = second
        A.append(w); b.append(cap)
        obj = np.array([float(jm["variables"][v].get(jm["optimize"]) or 0.0) for v in names] + [0.0] * k)
        s = -1.0 if sense == "max" else 1.0
        c = s * obj
    res = linprog(c, A_ub=np.array(A) if A else None, b_ub=np.array(b) if b else None, bounds=(0, None),
                  method="highs")
    if res.status == 2:
        return None
    if res.status == 3:
        return -s * math.inf
    assert res.status == 0, res.message
    return s * res.fun


def _close(a, b, tol=1e-7):
    if math.isinf(a) or math.isinf(b):
        return a == b
    return abs(a - b) <= tol * max(1.0, abs(a), abs(b))


def check(jm, weights=None, gap=0.0, absolute_gap=0.0):
    """The restatement of jm against HiGHS; returns (result, details)."""
    jm = strip_timeouts(jm)
    res, det = RO.repair(jm, weights, gap=gap, absolute_gap=absolute_gap)
    if res["stop"] == "cycled" and res["violation"] is None:
        return res, det
    want = highs_elastic(jm, det["rows"], det["weights"])
    if not res["feasible"]:
        assert want is None, ("HiGHS repairs a model the restatement calls infeasible", want)
        return res, det
    vstar = res["stages"][0]["optimum"]
    assert want is not None and _close(vstar, want), (vstar, want)
    # the plan meets every row, repaired ones at their repaired right-hand side
    names, R = _rows(jm)
    x = np.array([res["values"][v] for v in names])
    repaired = {(c["name"], c["type"]): c["repairedRhs"] for c in res["constraints"]}
    scale = max(1.0, float(np.abs(x).max(initial=0.0)))
    for cname, kind, a, rhs in R:
        b = repaired.get((cname, kind), rhs)
        tol = 1e-7 * max(1.0, abs(b)) * scale
        assert (a @ x <= b + tol) if kind == "max" else (a @ x >= b - tol), (cname, kind, a @ x, b)
    assert (x >= -1e-9 * scale).all()
    if res["stop"] == "reached":
        assert res["violation"] <= vstar + res["stages"][-1].get("allowance", 0.0) + 1e-7 * max(1.0, vstar)
    return res, det


def repaired_model(jm, res):
    """jm with every violated row's right-hand side moved to its repairedRhs."""
    cons = {k: dict(v) for k, v in jm["constraints"].items()}
    for c in res["constraints"]:
        spec = cons[c["name"]]
        if spec.get("equal") is not None:  # an equality relaxed on one side keeps the other
            lo = hi = spec.pop("equal")
            spec.update(min=lo, max=hi)
        spec[c["type"]] = c["repairedRhs"]
    return dict(jm, constraints=cons)


# ---------------------------------------------------------------- V* against HiGHS
@pytest.mark.parametrize("fx", INFEASIBLE, ids=lambda f: f["file"])
def test_infeasible_fixtures_match_highs(fx):
    pytest.importorskip("scipy")
    res, det = check(fx["model"])
    if res["stop"] == "cycled":
        pytest.skip("stage 1 cycles")
    assert res["feasible"] and res["stages"][0]["optimum"] > P and det["s1"][1] == 0


def test_planted_conflicts_unit_and_weighted():
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    for seed in range(3):
        jm = problems.planted_infeasible_model(14, 10, 3 + seed, seed=seed)
        res, det = check(jm)
        assert res["stages"][0]["optimum"] == 1.0 and res["violation"] == 1.0
        # weights: the conflict rows are p_j <= 1 (j < k-1) and sum p_j >= k; any one of them can absorb the unit
        names = [n for n in jm["constraints"] if n.startswith("conflict")]
        weights = {n: 5.0 + i for i, n in enumerate(names)}
        weights[names[1]] = 2.0  # the cheapest row
        res, det = check(jm, weights)
        assert res["stages"][0]["optimum"] == 2.0, res
        assert [c["name"] for c in res["constraints"]] == [names[1]] and res["constraints"][0]["violation"] == 1.0


def test_infeasible_packing_and_mixed_models_match_highs():
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    for seed in range(3):
        jm = problems.infeasible_packing_model(12 + seed, 10 + seed, 3 + seed, seed=seed)
        res, det = check(jm)
        assert len(det["crashed"]) == 3 + seed and det["s1"][1] == 0
        assert res["stages"][0]["crashed"] == 3 + seed
    seen = 0
    for k in range(20):
        jm = problems.mixed_lp_model(9, 8, seed=900 + k)
        res, det = check(jm)
        seen += res["feasible"]
    assert seen >= 10


def test_random_weights_and_subsets_match_highs():
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    rng = np.random.default_rng(7)
    jm = problems.infeasible_packing_model(10, 12, 4, seed=11)
    names = list(jm["constraints"])
    for _ in range(3):
        check(jm, {n: float(rng.uniform(0.1, 10.0)) for n in names})
    demand = [n for n in names if "min" in jm["constraints"][n]]
    packing = [n for n in names if "max" in jm["constraints"][n]]
    res, _ = check(jm, {n: 1.0 for n in demand})
    assert res["feasible"] and {c["type"] for c in res["constraints"]} == {"min"}
    res, _ = check(jm, {n: 2.0 for n in packing})  # only packing rows: still repairable, they absorb the demand
    assert res["feasible"]
    res, det = check(jm, {demand[0]: 1.0})  # the other demand rows cannot be relaxed
    assert not res["feasible"] and res["stop"] == "infeasible" and res["values"] is None
    # the side syntax on an equality: only its `min` row may move
    eq = {"optimize": "z", "opType": "max", "constraints": {"e": {"equal": 5}, "cap": {"max": 3}},
          "variables": {"x": {"z": 1, "e": 1, "cap": 1}}}
    res, det = check(eq, {"e": {"min": 3.0}})
    assert res["constraints"] == [{"name": "e", "type": "min", "rhs": 5, "weight": 3.0, "violation": 2.0,
                                   "repairedRhs": 3.0}]
    res, _ = check(eq, {"e": {"max": 3.0}})
    assert not res["feasible"]
    res, _ = check(eq, {"cap": 1.0})
    assert res["constraints"][0]["name"] == "cap" and res["constraints"][0]["repairedRhs"] == 5.0


def test_repaired_model_is_feasible():
    pytest.importorskip("scipy")
    from scipy.optimize import linprog
    from jslpsolver_b200 import problems
    cases = [BROKEN, problems.planted_infeasible_model(12, 9, 3, seed=2),
             problems.infeasible_packing_model(10, 10, 3, seed=4)] + [f["model"] for f in INFEASIBLE[:3]]
    for jm in cases:
        jm = strip_timeouts(jm)
        res, _ = RO.repair(jm)
        if res["violation"] is None:
            continue
        # the repaired right-hand sides sit exactly on the plan: loosen them by the precision they were read with
        fixed = repaired_model(jm, res)
        for spec in fixed["constraints"].values():
            if spec.get("min") is not None:
                spec["min"] -= 1e-7 * max(1.0, abs(spec["min"]))
            if spec.get("max") is not None:
                spec["max"] += 1e-7 * max(1.0, abs(spec["max"]))
        names, R = _rows(fixed)
        A = [a if kind == "max" else -a for _, kind, a, _ in R]
        b = [rhs if kind == "max" else -rhs for _, kind, _, rhs in R]
        out = linprog(np.zeros(len(names)), A_ub=np.array(A), b_ub=np.array(b), bounds=(0, None), method="highs")
        assert out.status == 0, (jm.get("name"), out.message)


def test_every_iis_holds_a_violated_row():
    """Cross-check against section 2c: a repair that left some IIS intact would not be feasible."""
    from jslpsolver_b200 import problems
    from oracle import iis as OI
    cases = [BROKEN, problems.planted_infeasible_model(12, 9, 3, seed=5),
             problems.infeasible_packing_model(8, 8, 2, seed=3)] + [f["model"] for f in INFEASIBLE]
    checked = 0
    for jm in cases:
        jm = strip_timeouts(jm)
        res, det = RO.repair(jm)
        if res["violation"] is None:
            continue
        M, vrow, vcol = det["M"], det["vrow"], det["vcol"]
        S0 = OI.start_set(M, vrow, vcol, None, P)[0]
        if S0 is None:
            continue
        kept = OI.literal_filter(M, vrow, vcol, None, P, S0)[0]
        e_of = dict(zip(det["rows"], det["e"]))
        assert any(e_of[r] > P for r in kept), (jm.get("name"), kept, e_of)
        checked += 1
    assert checked >= 4


# ---------------------------------------------------------------- stage 2
def test_stage_two_matches_highs_and_is_monotone():
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    cases = [BROKEN, problems.infeasible_packing_model(12, 12, 3, seed=21),
             problems.planted_infeasible_model(12, 9, 3, seed=8)]
    for jm in cases:
        prev = None
        sense = jm.get("opType", "min")
        for gap, absolute_gap in ((0.0, 0.0), (0.01, 0.0), (0.1, 0.0), (0.0, 5.0), (1.0, 0.0)):
            res, det = check(jm, gap=gap, absolute_gap=absolute_gap)
            vstar, s2 = res["stages"][0]["optimum"], res["stages"][1]
            want = highs_elastic(jm, det["rows"], det["weights"], (vstar + s2["allowance"], sense))
            z = s2["optimum"]
            assert _close(z, want), (gap, absolute_gap, z, want)
            assert _close(res["result"], z)
            if det["s2"] is not None:
                assert det["s2"][1] == 0, "stage 2 made a phase-1 pivot"
            if prev is not None and s2["allowance"] >= prev[0]:
                assert (z >= prev[1] - 1e-9 * max(1.0, abs(prev[1]))) if sense == "max" else \
                    (z <= prev[1] + 1e-9 * max(1.0, abs(prev[1])))
            prev = (s2["allowance"], z)
    res, _ = RO.repair(BROKEN)  # the README example: V* = 13 and the Berlin optimum survives
    assert res["violation"] == 13.0 and res["result"] == 1080000.0
    assert res["values"] == {"brit": 24.0, "yank": 20.0} and res["constraints"][0]["repairedRhs"] == 0.0


def test_unbounded_stage_two_keeps_the_stage_one_plan():
    jm = {"optimize": "z", "opType": "max", "constraints": {"need": {"min": 4}, "cap": {"max": 1}},
          "variables": {"x": {"z": 1, "need": 1, "cap": 1}, "y": {"z": 1}}}
    res, det = RO.repair(jm)
    assert res["stop"] == "unbounded" and res["stages"][0]["optimum"] == 3.0
    assert res["values"] == {"x": 1.0, "y": 0.0} and res["violation"] == 3.0


def test_feasible_model_repairs_to_its_optimum():
    from jslpsolver_b200 import problems
    from oracle import ref_model
    for jm in (BERLIN, problems.dense_packing_lp_model(12, 9, seed=3), problems.alternative_optima_model(14, 8, seed=2)):
        res, det = RO.repair(jm)
        assert res["violation"] == 0.0 and res["constraints"] == [] and res["stages"][0]["crashed"] == 0
        want = ref_model.Solve(jm)["result"]
        assert abs(res["result"] - want) <= 1e-6 * max(1.0, abs(want)), (res["result"], want)
        assert det["s1"][1] == 0 and det["s1"][2] == 0
    res, _ = RO.repair(BERLIN, objective=False)
    assert len(res["stages"]) == 1 and res["values"] == {"brit": 0.0, "yank": 0.0} and res["result"] == 0.0


# ---------------------------------------------------------------- rule 1
def test_row_zero_is_the_fixed_order_sum():
    """Rule 1 on a tableau with more crashed rows than one tile, weights that do not add exactly, and signed zeros."""
    rng = np.random.default_rng(3)
    H, W = 2 + 3 * RO.ELASTIC_TILE_ROWS, 9
    M = rng.normal(size=(H, W))
    M[0] = 0.0
    M[5, 3], M[6, 3] = 0.0, -0.0
    M[1:, 0] = np.where(rng.random(H - 1) < 0.7, -rng.uniform(0.5, 2.0, H - 1), rng.uniform(0.5, 2.0, H - 1))
    M[7, 0], M[8, 0] = -P, -np.nextafter(P, 1.0)  # at -P: not crashed; one ulp below: crashed
    vrow = np.arange(-1, H - 1, dtype=np.int32)
    vcol = np.concatenate([[-1], np.arange(H - 1, H + W - 2)]).astype(np.int32)
    rows = [r for r in range(1, H) if r % 5]
    w = list(rng.uniform(0.1, 3.0, len(rows)))
    E, vr, vc, crashed = RO.elastic(M, vrow, vcol, P, rows, w, H + W - 2)
    assert 7 not in crashed and 8 in crashed
    bits = lambda a: np.ascontiguousarray(a).view(np.uint64)  # noqa: E731
    want = np.zeros(W + len(rows))
    for t0 in range(1, H, RO.ELASTIC_TILE_ROWS):
        part = np.zeros(W + len(rows))
        for r in range(t0, min(H, t0 + RO.ELASTIC_TILE_ROWS)):
            if r in crashed:
                part = part + w[rows.index(r)] * E[r]
        want = want + part
    for j, r in enumerate(rows):
        if r not in crashed:
            want[W + j] = -w[j]
        assert E[r, W + j] == -1.0 and (E[r, W:] != 0).sum() == 1
    assert np.array_equal(bits(E[0]), bits(want))
    for r in range(1, H):
        if r in crashed:
            assert np.array_equal(bits(E[r, :W]), bits(M[r]) ^ RO.SIGN_BIT) and vr[r] == H + W - 2 + rows.index(r)
        else:
            assert np.array_equal(bits(E[r, :W]), bits(M[r])) and vr[r] == vrow[r]
    assert np.signbit(E[5, 3]) == (5 in crashed) and np.signbit(E[6, 3]) == (6 not in crashed)


# ---------------------------------------------------------------- the host driver over a stand-in tableau
class _Stub:
    """Stands in for GpuTableau over the restatement: upload, elastic (rule 1), simplex, lex_next (rule 3)."""

    def __init__(self, log, M=None, vrow=None, vcol=None, n=0):
        self.log, self.M, self.vrow, self.vcol, self.nVars = log, M, vrow, vcol, n
        self.closed = False
        log.append(self)
        self.feasible = self.bounded = True

    @property
    def width(self):
        return self.M.shape[1]

    @property
    def height(self):
        return self.M.shape[0]

    def upload(self, M, vrow, vcol, unrestricted=None):
        self.M, self.vrow, self.vcol = np.array(M), np.array(vrow), np.array(vcol)
        self.nVars = M.shape[0] + M.shape[1] - 2

    def elastic(self, rows, weights):
        E, vr, vc, crashed = RO.elastic(self.M, self.vrow, self.vcol, P, list(rows), list(weights), self.nVars)
        return _Stub(self.log, E, vr, vc, self.nVars + len(rows)), len(crashed)

    def lex_next(self, cost, t):
        assert not self.closed and len(cost) == self.nVars
        import lexicographic_oracle as LO
        T, vr, vc, kept = LO.child(self.M, self.vrow, self.vcol, P, np.asarray(cost, dtype=np.float64), t, self.nVars)
        if T is None:
            return None, kept
        return _Stub(self.log, T, vr, vc, self.nVars + (t > 0.0)), kept

    def simplex(self, check_cycles=None):
        assert check_cycles is True
        import lexicographic_oracle as LO
        status, p1, p2, self.M, self.vrow, self.vcol = LO.solve(self.M, self.vrow, self.vcol, P)
        self.lastStatus = types.SimpleNamespace(phase1_pivots=p1, phase2_pivots=p2, cycled=int(status == LO.CYCLED))
        self.feasible, self.bounded = status != LO.INFEASIBLE, status != LO.UNBOUNDED
        return self

    def final_state(self):
        return self.M[:, 0].copy(), self.M[0].copy(), self.vrow, self.vcol

    def close(self):
        self.closed = True


class _StubSolver:
    def __init__(self):
        self.log = []

    def _instance(self, model, precision):
        import jslpsolver_b200.tableau as T
        from jslpsolver_b200.model import Model
        saved = T.GpuTableau
        T.GpuTableau = lambda *a, **k: None
        try:
            m = Model(precision).loadJson(model)
        finally:
            T.GpuTableau = saved
        m.tableau = _Stub(self.log)
        return m


def test_host_driver_equals_the_restatement():
    from jslpsolver_b200 import problems
    from jslpsolver_b200.repair import Repair
    eq = {"optimize": "z", "opType": "max", "constraints": {"e": {"equal": 5}, "cap": {"max": 3}},
          "variables": {"x": {"z": 1, "e": 1, "cap": 1}}}
    ray = {"optimize": "z", "opType": "max", "constraints": {"need": {"min": 4}, "cap": {"max": 1}},
           "variables": {"x": {"z": 1, "need": 1, "cap": 1}, "y": {"z": 1}}}
    cases = [(BROKEN, {}), (BROKEN, {"gap": 0.1}), (BROKEN, {"objective": False}), (BERLIN, {}), (ray, {}),
             (eq, {"weights": {"e": {"min": 3.0}}}), (eq, {"weights": {"e": {"max": 3}}}),
             (dict(BROKEN, optimize={"capacity": "max"}), {"absolute_gap": 2.0}),
             (problems.infeasible_packing_model(10, 10, 3, seed=1), {"weights": {"c1": 2.0, "c4": 0.5}}),
             (problems.infeasible_packing_model(10, 10, 3, seed=2), {"gap": 0.05}),
             (problems.planted_infeasible_model(10, 8, 3, seed=3), {})]
    for jm, kw in cases:
        s = _StubSolver()
        got = Repair(s, jm, **kw)
        want, _ = RO.repair(jm, kw.get("weights"), kw.get("objective", True), kw.get("gap", 0.0),
                            kw.get("absolute_gap", 0.0))
        assert got == want, (kw, got, want)
        assert len(s.log) == 2 + (len(got["stages"]) > 1 and got["stages"][1]["width"] is not None)
        assert all(t.closed for t in s.log), "a scratch tableau was left open"


def test_refusals_and_weight_errors():
    from jslpsolver_b200.repair import Repair
    s = _StubSolver()
    for model, match in ((dict(BERLIN, ints={"brit": 1}), "integer or binary"),
                         (dict(BERLIN, binaries={"yank": 1}), "integer or binary"),
                         (dict(BERLIN, constraints=dict(BERLIN["constraints"], plane={"max": 44, "weight": 3})), "soft"),
                         (dict(BERLIN, constraints=dict(BERLIN["constraints"], plane={"max": 44, "priority": 1})), "soft"),
                         (dict(BERLIN, unrestricted={"brit": 1}), "unrestricted variables"),
                         (dict(BERLIN, optimize={"capacity": "max", "cost": "min"}), "one objective"),
                         (dict(BERLIN, external={"solver": "x"}), "external")):
        with pytest.raises(ValueError, match=r"Repair\(\).*" + re.escape(match)):
            Repair(s, model)
    for weights, match in (({"nope": 1.0}, "no constraint named 'nope'"), ({"plane": 0.0}, "must be finite and > 0"),
                           ({"plane": -1}, "must be finite and > 0"), ({"plane": math.nan}, "finite and > 0"),
                           ({"plane": math.inf}, "finite and > 0"), ({"plane": True}, "must be a number"),
                           ({"plane": "1"}, "must be a number"), ({"plane": None}, "must be a number"),
                           ({"plane": {}}, "needs a 'min'"), ({"plane": {"equal": 1}}, "side must be"),
                           ({"plane": {"min": 1.0}}, "only a 'max' bound"), ({"plane": {"max": 0}}, "finite and > 0"),
                           ([1.0], "takes a dict")):
        with pytest.raises(ValueError, match=r"Repair\(\).*" + re.escape(match)):
            Repair(s, BROKEN, weights)
    for kw, match in (({"gap": -0.1}, "gap= must be finite and >= 0"), ({"absolute_gap": math.nan}, "absolute_gap="),
                      ({"gap": True}, "gap= takes a number")):
        with pytest.raises(ValueError, match=r"Repair\(\).*" + re.escape(match)):
            Repair(s, BROKEN, **kw)
    assert all(t.M is None for t in s.log), "a refused call uploaded a tableau"
    wide = {"optimize": "z", "opType": "max", "constraints": {f"r{i}": {"max": 1} for i in range(25599)},
            "variables": {"x": {"z": 1, **{f"r{i}": 1 for i in range(25599)}}}}
    with pytest.raises(ValueError, match=r"Repair\(\): the elastic tableau needs 25601 columns .*cap of 25600"):
        Repair(s, wide)
    assert all(t.M is None for t in s.log)
    wide["constraints"].pop("r0")
    assert Repair(s, wide, {"r1": 1.0})["violation"] == 0.0  # 2 + 1 columns: well inside the cap


def test_ctypes_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    import jslpsolver_b200 as J
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+jslp_elastic_create\s*\(([^)]*)\)\s*;", header)
    assert proto, "jslp_elastic_create is not declared"
    params = [re.sub(r"\s+", " ", p.strip()) for p in proto.group(1).split(",")]
    types_ = [re.sub(r"\s*\b\w+$", "", p).replace(" *", "*") for p in params]
    assert types_ == ["jslp_tab*", "const int32_t*", "const double*", "int", "jslp_tab**", "int32_t*"], types_
    assert "section 2k" in header[:proto.start()][-1500:]
    (name, res, args), = [s for s in _lib.SYMBOLS if s[0] == "jslp_elastic_create"]
    C = _lib.C
    assert res is C.c_int and len(args) == 6 and args[0] is C.c_void_p and args[1] is C.c_void_p
    assert args[2] is C.c_void_p and args[3] is C.c_int and args[4]._type_ is C.c_void_p
    assert args[5]._type_ is C.c_int32
    src = open(os.path.join(ROOT, "jslpsolver_b200", "csrc", "jslp_api.cu")).read()
    assert '#include "jslp_elastic.cuh"' in src.split('#include "jslp_lex.cuh"')[1]
    from jslpsolver_b200 import build
    assert any(d.endswith("jslp_elastic.cuh") for d in build.DEPS)
    assert J.Repair is not None and J.Solver.Repair is not None and "Repair" in J.__all__

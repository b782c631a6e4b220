"""CPU checks of near-optimal variability (DESIGN.md section 2i): Solution.variability(gap=..., absolute_gap=...) over
the restatement in near_optimal_oracle.py against SciPy HiGHS -- for every target, the min and max of the variable or
row slack subject to the model's constraints plus `objective >= z - t` (max) / `<= z + t` (min) -- on the fixtures,
seeded LPs, a presolve-fixed variable and an unbounded near-optimal set; nesting in t, the exact ranges inside the
near-optimal ones, the feasible set's ranges at a huge allowance, feasible argmin / argmax points within t of z; the
bound tableau at its sign-flip cases; t == 0 being the section 2h report; every ValueError; and the C prototype."""
import math
import os
import re

import numpy as np
import pytest

import near_optimal_oracle as NO
import test_variability_cpu as TV
from conftest import ROOT, load_bundle
from helpers import strip_timeouts

BUNDLE = load_bundle()
P = 1e-8


class _Stub(TV._StubTableau):
    """TV's stand-in for GpuTableau over the solved oracle tableau, plus bound(): the restated bound tableau, whose
    targets the stand-in batch runs through oracle/variability.target as the device batch would."""

    def __init__(self, model, sol):
        super().__init__(model, sol)
        self.bounds = []

    def bound(self, t):
        M, (vrow, vcol) = self.sol.tableau.matrix(), self.sol.tableau.maps()
        n = M.shape[0] + M.shape[1] - 2  # a fresh upload's n_index and lastElementIndex
        B, vrow_b, vcol_b = NO.bound(M, vrow, vcol, t, NO.fresh_label(n, n))
        self.bounds.append(t)
        self.faces.append(TV._StubFace(self, B, vrow_b, vcol_b))
        return self.faces[-1]


def _solution(jm, feasible=None, bounded=None):
    from jslpsolver_b200.tableau import Solution
    from oracle import ref_model
    sol = ref_model.solve_full(jm, fast_cycles=True)
    t = _Stub(TV._cpu_model(jm), sol)
    return Solution(t, sol.evaluation, sol.feasible if feasible is None else feasible,
                    sol.bounded if bounded is None else bounded)


class _Highs(TV._Highs):
    """TV's HiGHS model with the objective bound `c.x >= z - t` (max) / `c.x <= z + t` (min) in place of `c.x = z`;
    t = None drops the objective altogether (the feasible set)."""

    def __init__(self, jm, t):
        super().__init__(jm)
        self.t = t

    def extreme(self, expr, const, sense):
        A, b = self.A, self.b
        if self.t is not None:  # kappa * c.x <= kappa * z + t, kappa = -1 for max
            A = np.vstack([A, self.kappa * self.c[None, :]])
            b = np.append(b, self.kappa * self.z + self.t)
        res = self.linprog(-sense * expr, A_ub=A, b_ub=b, bounds=(0, None), method="highs")
        if res.status == 3:
            return sense * math.inf
        assert res.status == 0, res.message
        return -sense * res.fun + const

    def check_point(self, point, tol=1e-7):
        x = np.array([point[v] for v in self.names])
        scale = max(1.0, float(np.abs(x).max(initial=0.0)))
        assert (x >= -tol * scale).all(), point
        assert (self.A @ x <= self.b + tol * np.maximum(1.0, np.abs(self.b)) * scale).all(), point
        loss = -self.kappa * (self.z - float(self.c @ x))  # what the point gives up against the optimum
        assert loss <= self.t + tol * max(1.0, abs(self.z)), (loss, self.t)


def _check_against_highs(jm, gap=0.0, absolute_gap=0.0, variables=None, constraints=None):
    """Solution.variability(gap, absolute_gap, points=True) of jm over the restatement against HiGHS; returns the report
    (None: no optimum)."""
    jm = strip_timeouts(jm)
    sol = _solution(jm)
    if sol._tableau.sol.tableau is None or not (sol.feasible and sol.bounded):
        return None
    v = sol.variability(variables=variables, constraints=constraints, points=True, gap=gap, absolute_gap=absolute_gap)
    t = sol._tableau
    M, (vrow, vcol) = t.sol.tableau.matrix(), t.sol.tableau.maps()
    want_t = NO.allowance(gap, absolute_gap, M[0, 0])
    assert want_t > 0 and v["allowance"] == want_t and t.bounds == [want_t]
    assert v["free"] == M.shape[1] - 1 and v["lps"] == len(t.targets) and t.batches == (1 if v["lps"] else 0)
    assert all(f.closed for f in t.faces), "the bound tableau was not closed"
    basic = {int(x) for x in vrow[1:]}
    assert v["lps"] == sum(2 if lab in basic else 1 for lab in dict.fromkeys(lab for lab, _ in t.targets))
    h = _Highs(jm, want_t)
    assert h.status == 0
    if not v["exact"]:
        return v
    tol = lambda x: 1e-6 * max(1.0, abs(x))  # noqa: E731
    for vid, e in v["variables"].items():
        for side, s in (("min", -1), ("max", 1)):
            assert TV._close(e[side], h.variable(vid, s)), (vid, side, e[side], h.variable(vid, s))
            if e["arg" + side] is not None and not math.isinf(e[side]):
                h.check_point(e["arg" + side])
                assert TV._close(e["arg" + side][vid], e[side]), (vid, side, e)
        assert e["min"] - tol(e["value"]) <= e["value"] <= e["max"] + tol(e["value"]), (vid, e)
    for c in v["constraints"]:
        e = c["slack"]
        for side, s in (("min", -1), ("max", 1)):
            want = h.slack(c["name"], c["type"], s)
            assert TV._close(e[side], want), (c["name"], c["type"], side, e, want)
            if e["arg" + side] is not None and not math.isinf(e[side]):
                h.check_point(e["arg" + side])
    return v


@pytest.mark.parametrize("fx", [f for f in TV.CONTINUOUS if f["file"] != "Monster Problem.json"],
                         ids=lambda f: f["file"])
def test_fixture_ranges_match_highs(fx):
    pytest.importorskip("scipy")
    if _check_against_highs(fx["model"], gap=0.01) is None:
        pytest.skip("no optimum")


def test_monster_problem_sampled():
    """The 600-row fixture: the restatement's ranges of every 40th variable and row against HiGHS (the report itself
    would run an LP for every structural variable)."""
    pytest.importorskip("scipy")
    jm = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Monster Problem.json"][0]["model"])
    sol = _solution(jm)
    M, (vrow, vcol) = sol._tableau.sol.tableau.matrix(), sol._tableau.sol.tableau.maps()
    m = sol._tableau.model
    t = NO.allowance(0.002, 0.0, M[0, 0])
    n = M.shape[0] + M.shape[1] - 2
    vs, cs = m.variables[::40], [c for c in m.constraints][::40]
    want, free, lps, _ = NO.ranges(M, vrow, vcol, P, [x.index for x in vs] + [c.index for c in cs], t,
                                   NO.fresh_label(n, n))
    assert free == M.shape[1] - 1 and lps >= len(vs) + len(cs)
    h = _Highs(jm, t)
    for x in vs:
        for side, s in (("min", -1), ("max", 1)):
            assert TV._close(want[x.index][side], h.variable(x.id, s)), (x.id, side, want[x.index][side])
    for c in cs:
        kind = "max" if c.isUpperBound else "min"
        for side, s in (("min", -1), ("max", 1)):
            assert TV._close(want[c.index][side], h.slack(c.name, kind, s)), (c.name, side, want[c.index][side])


@pytest.mark.parametrize("gap,absolute_gap", [(1e-3, 0.0), (0.02, 0.0), (0.0, 5.0), (0.01, 40.0), (0.25, 0.0)])
def test_planted_and_seeded_lps_match_highs(gap, absolute_gap):
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    for seed in range(2):
        v = _check_against_highs(problems.alternative_optima_model(16 + seed, 8 + seed, seed=60 + seed), gap, absolute_gap)
        assert v["exact"] and not v["unique"]
        assert _check_against_highs(problems.dense_packing_lp_model(12 + seed, 9 + seed, seed=70 + seed), gap,
                                    absolute_gap) is not None
    checked = 0
    for k in range(30):
        v = _check_against_highs(problems.mixed_lp_model(10, 8, seed=800 + k), gap, absolute_gap)
        checked += v is not None and v["exact"]
        if checked >= 2:
            return
    pytest.fail(f"only {checked} seeded mixed LPs had an optimum")


def test_presolve_fixed_variable():
    """-x <= -2 and x <= 2: presolve fixes x = 2 (no LP, [2, 2]); y and w share `cap` and may now give up objective."""
    pytest.importorskip("scipy")
    v = _check_against_highs(TV.FIXED, absolute_gap=3.0)
    assert v["variables"]["x"] == dict(v["variables"]["x"], value=2, min=2, max=2, fixed=True)
    assert (v["variables"]["y"]["min"], v["variables"]["y"]["max"]) == (0.0, 5.0)
    sol = _solution(TV.FIXED)
    sol.variability(absolute_gap=3.0)
    x = next(u for u in sol._tableau.model.variables if u.id == "x").index
    assert all(lab != x for lab, _ in sol._tableau.targets)


def test_unbounded_near_optimal_set():
    """max x, x - y <= 2, x <= 5: the optimum pins x = 5 and lets y run off (y >= 3); with the allowance x may drop."""
    pytest.importorskip("scipy")
    jm = {"optimize": "z", "opType": "max", "constraints": {"gap": {"max": 2}, "cap": {"max": 5}},
          "variables": {"x": {"z": 1, "gap": 1, "cap": 1}, "y": {"gap": -1}}}
    v = _check_against_highs(jm, absolute_gap=1.5)
    assert v["exact"] and v["allowance"] == 1.5
    assert (v["variables"]["x"]["min"], v["variables"]["x"]["max"]) == (3.5, 5.0)
    assert v["variables"]["y"]["max"] == math.inf and v["variables"]["y"]["argmax"] is None
    assert v["variables"]["y"]["min"] == 1.5
    ray = {"optimize": "z", "opType": "max", "constraints": {"gap": {"max": 2}, "low": {"min": 1}},
           "variables": {"x": {"z": 1, "gap": 1, "low": 1}, "y": {"z": -1, "gap": -1}}}
    w = _check_against_highs(ray, gap=0.5)
    assert w["variables"]["x"]["max"] == math.inf and w["variables"]["x"]["min"] == 1.0


def test_properties_nesting_exact_inside_and_feasible_set():
    """Ranges grow with t, the section 2h ranges lie inside every near-optimal one, and an allowance beyond any loss
    gives the ranges over the feasible set alone."""
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    jm = problems.alternative_optima_model(18, 10, seed=5)
    sol = _solution(jm)
    exact = sol.variability()
    reports = [sol.variability(gap=g) for g in (1e-4, 1e-2, 0.1)] + [sol.variability(absolute_gap=1e9)]
    eps = lambda x: 1e-9 * max(1.0, abs(x))  # noqa: E731
    for inner, outer in zip([exact] + reports, reports):
        for vid in exact["variables"]:
            a, b = inner["variables"][vid], outer["variables"][vid]
            assert b["min"] <= a["min"] + eps(a["min"]) and a["max"] <= b["max"] + eps(a["max"]), (vid, a, b)
        for a, b in zip(inner["constraints"], outer["constraints"]):
            a, b = a["slack"], b["slack"]
            assert b["min"] <= a["min"] + eps(a["min"]) and a["max"] <= b["max"] + eps(a["max"]), (a, b)
    h = _Highs(jm, None)
    assert h.status == 0
    huge = reports[-1]
    for vid, e in huge["variables"].items():
        assert TV._close(e["min"], h.variable(vid, -1)) and TV._close(e["max"], h.variable(vid, 1)), (vid, e)
    assert not huge["unique"] and huge["allowance"] == 1e9


def test_zero_allowance_is_the_exact_report():
    """t == 0 takes the face path: the section 2h report key for key and bit for bit, no bound tableau, no
    "allowance"; also when z == 0 and only gap is set."""
    from jslpsolver_b200 import problems
    for jm in (problems.alternative_optima_model(16, 8, seed=2), TV.HAND, TV.BERLIN):
        a, b = _solution(jm), _solution(jm)
        want = a.variability(points=True)
        for kw in ({}, {"gap": 0.0}, {"absolute_gap": 0}, {"gap": 0.0, "absolute_gap": 0.0}):
            got = b.variability(points=True, **kw)
            assert got == want and list(got) == list(want) and "allowance" not in got
        assert b._tableau.bounds == [] and a._tableau.targets * 4 == b._tableau.targets
    zero = {"optimize": "cost", "opType": "min", "constraints": {"cap": {"max": 4}, "need": {"min": 0}},
            "variables": {"x": {"cost": 1, "cap": 1, "need": 1}, "y": {"cost": 2, "cap": 1}}}
    s = _solution(zero)
    assert s._tableau.sol.tableau.matrix()[0, 0] == 0 and s.evaluation == 0
    assert s.variability(gap=0.5) == s.variability() and s._tableau.bounds == []
    assert s.variability(gap=0.5, absolute_gap=1.0)["allowance"] == 1.0


def test_bound_tableau_rule_at_its_sign_cases():
    """Rule 1: rows 1..H-1 bit for bit, row 0 +0, B[H,0] = t and B[H,c] = -M[0,c] as a sign flip (+0 -> -0, -0 -> +0,
    +-P, NaN payloads kept), vrow' = (vrow, l*), vcol' = vcol."""
    cost = [123.0, P, -P, 0.0, -0.0, math.nan, -math.nan, 5.0, -5.0, 1e-300, math.inf, -math.inf]
    M = np.arange(3 * len(cost), dtype=np.float64).reshape(3, len(cost)) - 7.5
    M[0] = cost
    M[2, 3], M[1, 5] = -0.0, math.nan
    vrow, vcol = np.array([-1, 20, 21], dtype=np.int32), np.arange(100, 100 + len(cost), dtype=np.int32)
    B, vrow_b, vcol_b = NO.bound(M, vrow, vcol, 2.5, 777)
    bits = lambda a: np.ascontiguousarray(a).view(np.uint64)  # noqa: E731
    assert B.shape == (4, len(cost)) and not np.signbit(B[0]).any() and (B[0] == 0).all()
    assert np.array_equal(bits(B[1:3]), bits(M[1:3]))
    assert B[3, 0] == 2.5 and np.array_equal(bits(B[3, 1:]), bits(M[0, 1:]) ^ NO.SIGN_BIT)
    assert np.signbit(B[3, 3]) and not np.signbit(B[3, 4]) and math.isnan(B[3, 5]) and B[3, 1] == -P
    assert list(vrow_b) == [-1, 20, 21, 777] and np.array_equal(vcol_b, vcol)
    assert NO.fresh_label(10, 12) == 12 and NO.fresh_label(10, 10) == 10
    assert NO.allowance(0.01, 0.0, -250.0) == 2.5 and NO.allowance(0.01, 7.0, 250.0) == 7.0


def test_every_non_basic_label_runs_one_lp():
    """Rule 3: two LPs per basic label, one (the max) per non-basic label, none for a presolve-fixed variable; the
    submission order is section 2h's, and variables= / constraints= restrict the report, not the variables."""
    from jslpsolver_b200 import problems
    jm = problems.alternative_optima_model(20, 10, seed=3)
    sol = _solution(jm)
    t, m = sol._tableau, sol._tableau.model
    M, (vrow, vcol) = t.sol.tableau.matrix(), t.sol.tableau.maps()
    basic = {int(x) for x in vrow[1:]}
    labels = [x.index for x in m.variables] + [c.index for c in m.constraints]
    v = sol.variability(gap=0.05)
    want_targets = [(lab, s) for lab in labels for s in ((-1, 1) if lab in basic else (1,))]
    assert t.targets == want_targets and v["lps"] == len(want_targets) and v["free"] == M.shape[1] - 1
    n = M.shape[0] + M.shape[1] - 2
    want, free, lps, submitted = NO.ranges(M, vrow, vcol, P, labels, v["allowance"], NO.fresh_label(n, n))
    assert (free, lps, submitted) == (v["free"], v["lps"], want_targets)
    for x in m.variables:
        assert (want[x.index]["min"], want[x.index]["max"]) == (v["variables"][x.id]["min"], v["variables"][x.id]["max"])
    t.targets.clear()
    part = sol.variability(variables=["x0"], constraints=["c1"], gap=0.05)
    assert list(part["variables"]) == ["x0"] and [c["name"] for c in part["constraints"]] == ["c1"]
    assert part["variables"]["x0"] == v["variables"]["x0"] and part["unique"] == v["unique"]
    assert [lab for lab, _ in t.targets] == [lab for lab, _ in want_targets
                                            if lab in {x.index for x in m.variables} or lab == m.constraints[1].index]


def test_value_errors():
    from jslpsolver_b200.tableau import Solution
    sol = _solution(TV.BERLIN)
    for kw, match in (({"gap": -0.01}, "gap= must be finite and >= 0"), ({"gap": math.nan}, "gap= must be finite"),
                      ({"gap": math.inf}, "gap= must be finite"), ({"absolute_gap": -1}, "absolute_gap= must be"),
                      ({"absolute_gap": math.nan}, "absolute_gap= must be"), ({"absolute_gap": -math.inf}, "absolute_gap="),
                      ({"gap": "1%"}, "gap= takes a number"), ({"gap": None}, "gap= takes a number"),
                      ({"absolute_gap": True}, "absolute_gap= takes a number"), ({"gap": [0.1]}, "gap= takes a number"),
                      ({"gap": 1e308}, "overflows"), ({"variables": ["nope"], "gap": 0.1}, "no variable named"),
                      ({"constraints": "plane", "gap": 0.1}, "takes a list")):
        with pytest.raises(ValueError, match=r"variability\(\).*" + re.escape(match)):
            sol.variability(**kw)
    assert sol._tableau.batches == 0 and sol._tableau.bounds == [], "a refused call ran LPs"
    assert sol.variability(gap=np.float64(0.01))["allowance"] == 0.01 * 1080000.0 == 10800.0
    free = dict(TV.BERLIN, unrestricted={"brit": 1})
    with pytest.raises(ValueError, match=r"variability\(\) does not support unrestricted variables"):
        _solution(free).variability(gap=0.01)
    lp0 = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Berlin Air Lift Problem.json"][0]["model"])
    mip = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Integer Berlin Air Lift Problem.json"][0]["model"])
    soft = dict(lp0, constraints=dict(lp0["constraints"], plane={"max": 44, "weight": 10}))
    for model, feasible, bounded, match in ((mip, True, True, "integer or binary"), (soft, True, True, "soft constraints"),
                                            (lp0, False, True, "infeasible"), (lp0, True, False, "unbounded")):
        with pytest.raises(ValueError, match=r"variability\(\).*" + match):
            _solution(model, feasible, bounded).variability(gap=0.01)
    s = _solution(lp0)
    s._tableau._version += 1
    with pytest.raises(ValueError, match="edited or solved again"):
        s.variability(absolute_gap=1.0)
    s._tableau.handle = None
    with pytest.raises(ValueError, match="has not been solved"):
        Solution(s._tableau, 0.0, True, True).variability(gap=0.01)


def test_ctypes_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+jslp_bound_create\s*\(([^)]*)\)\s*;", header)
    assert proto, "jslp_bound_create is not declared"
    params = [re.sub(r"\s+", " ", p.strip()) for p in proto.group(1).split(",")]
    types = [re.sub(r"\s*\b\w+$", "", p).replace(" *", "*") for p in params]
    assert types == ["jslp_tab*", "double", "jslp_tab**"], types
    assert "section 2i" in header[:proto.start()][-1500:]
    (name, res, args), = [s for s in _lib.SYMBOLS if s[0] == "jslp_bound_create"]
    C = _lib.C
    assert res is C.c_int and len(args) == 3 and args[0] is C.c_void_p and args[1] is C.c_double
    assert args[2]._type_ is C.c_void_p
    src = open(os.path.join(ROOT, "jslpsolver_b200", "csrc", "jslp_api.cu")).read()
    assert '#include "jslp_bound.cuh"' in src.split('#include "jslp_face.cuh"')[1]

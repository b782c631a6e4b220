"""CPU checks of alternative optima (DESIGN.md section 2h): Solution.variability() over the oracle definition against
SciPy HiGHS -- for every target, the min and max of the variable or row slack subject to the model's constraints plus
`objective = z*` -- on the fixtures, seeded LPs with planted alternative optima, an unbounded face and a presolve-fixed
variable; every argmin / argmax point is feasible and optimal; the face rules at their thresholds; the LP counts of
rule 4; the known answers; every ValueError; and the C prototype against the header."""
import math
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_bundle
from helpers import strip_timeouts

BUNDLE = load_bundle()
BERLIN = {"optimize": "capacity", "opType": "max",
          "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
          "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                        "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}
HAND = {"optimize": "profit", "opType": "max",
        "constraints": {"both": {"max": 4}, "capx": {"max": 3}, "capy": {"max": 3}},
        "variables": {"x": {"profit": 1, "both": 1, "capx": 1}, "y": {"profit": 1, "both": 1, "capy": 1}}}
FIXED = {"optimize": "z", "opType": "max", "constraints": {"lo": {"max": -2}, "hi": {"max": 2}, "cap": {"max": 7}},
         "variables": {"x": {"z": 1, "lo": -1, "hi": 1, "cap": 1}, "y": {"z": 2, "cap": 1}, "w": {"z": 2, "cap": 1}}}


def _soft(jm):
    return any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())


CONTINUOUS = [f for f in BUNDLE["fixtures"] + BUNDLE["readme"]
              if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"])
                      or f["model"].get("unrestricted"))
              and isinstance(f["model"].get("optimize"), str)]


def _cpu_model(jm):
    """The host Model of jm as Model.solve() leaves it (presolve applied), without a device tableau."""
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


class _StubFace:
    """Stands in for the face GpuTableau: runs the oracle definition of every target as the device batch would."""

    def __init__(self, owner, F, vrow, vcol_f):
        self.owner, self.F, self.vrow, self.vcol = owner, F, vrow, vcol_f
        self.closed = False

    def scenario_batch(self, edits, offsets, check_cycles=None):
        from oracle import variability as OV
        assert check_cycles is True and list(offsets) == list(range(len(edits) + 1))
        self.owner.batches += 1
        out = {k: [] for k in ("status", "eval_raw", "p1", "p2", "rhs", "vrow")}
        for kind, label, difference in edits:
            assert kind == 1 and difference in (1.0, -1.0)
            got = OV.target(self.F, self.vrow, self.vcol, self.owner.precision, label, -difference)
            for k, x in zip(out, got):
                out[k].append(x)
        self.owner.targets += [(label, int(-d)) for _, label, d in edits]
        return out

    def close(self):
        self.closed = True


class _StubTableau:
    """Stands in for GpuTableau over the solved oracle tableau."""

    def __init__(self, model, sol):
        self.model, self.sol = model, sol
        self.handle = object()
        self._version = self._solved_version = 0
        self.precision = model.precision
        self.variablesPerIndex = model.variablesPerIndex
        self.batches, self.targets, self.faces = 0, [], []

    def final_state(self):
        M, (vrow, vcol) = self.sol.tableau.matrix(), self.sol.tableau.maps()
        return M[:, 0].copy(), M[0].copy(), vrow, vcol

    def face(self):
        from oracle import variability as OV
        M, (vrow, vcol) = self.sol.tableau.matrix(), self.sol.tableau.maps()
        kept, F, vcol_f = OV.face(M, vcol, self.precision)
        if len(kept) == 1:
            return None, kept
        self.faces.append(_StubFace(self, F, vrow, vcol_f))
        return self.faces[-1], kept


def _solution(jm, feasible=None, bounded=None):
    from jslpsolver_b200.tableau import Solution
    from oracle import ref_model
    sol = ref_model.solve_full(jm, fast_cycles=True)
    t = _StubTableau(_cpu_model(jm), sol)
    return Solution(t, sol.evaluation, sol.feasible if feasible is None else feasible,
                    sol.bounded if bounded is None else bounded)


# ---------------------------------------------------------------- the HiGHS reference
def _rows(jm, names):
    """[(constraint name, 'max' | 'min', a, b)]: a.x <= b or a.x >= b."""
    out = []
    for cname, spec in jm["constraints"].items():
        a = np.array([jm["variables"][v].get(cname, 0.0) for v in names], dtype=np.float64)
        lo, hi = (spec["equal"], spec["equal"]) if spec.get("equal") is not None else (spec.get("min"), spec.get("max"))
        if hi is not None:
            out.append((cname, "max", a, float(hi)))
        if lo is not None:
            out.append((cname, "min", a, float(lo)))
    return out


class _Highs:
    def __init__(self, jm):
        from scipy.optimize import linprog
        self.linprog = linprog
        self.names = list(jm["variables"])
        self.rows = _rows(jm, self.names)
        self.kappa = -1.0 if jm.get("opType") == "max" else 1.0
        self.c = np.array([jm["variables"][v].get(jm["optimize"], 0.0) for v in self.names], dtype=np.float64)
        self.A = np.array([a if kind == "max" else -a for _, kind, a, _ in self.rows])
        self.b = np.array([b if kind == "max" else -b for _, kind, _, b in self.rows])
        res = linprog(self.kappa * self.c, A_ub=self.A, b_ub=self.b, bounds=(0, None), method="highs")
        self.status = res.status
        self.z = self.kappa * res.fun if res.status == 0 else None

    def extreme(self, expr, const, sense):
        """max (sense +1) or min (-1) of expr.x + const over the optimal face; +-inf when unbounded."""
        res = self.linprog(-sense * expr, A_ub=self.A, b_ub=self.b, A_eq=self.c[None, :], b_eq=[self.z],
                           bounds=(0, None), method="highs")
        if res.status == 3:
            return sense * math.inf
        assert res.status == 0, res.message
        return -sense * res.fun + const

    def variable(self, vid, sense):
        e = np.zeros(len(self.names))
        e[self.names.index(vid)] = 1.0
        return self.extreme(e, 0.0, sense)

    def slack(self, cname, kind, sense):
        (a, b), = [(a, b) for n, k, a, b in self.rows if n == cname and k == kind]
        return self.extreme(-a, b, sense) if kind == "max" else self.extreme(a, -b, sense)

    def check_point(self, point, tol=1e-7):
        x = np.array([point[v] for v in self.names])
        scale = max(1.0, float(np.abs(x).max(initial=0.0)))
        assert (x >= -tol * scale).all(), point
        assert (self.A @ x <= self.b + tol * np.maximum(1.0, np.abs(self.b)) * scale).all(), point
        assert abs(float(self.c @ x) - self.z) <= tol * max(1.0, abs(self.z)), (float(self.c @ x), self.z)


def _close(a, b, tol=1e-6):
    if a is None or b is None:
        return False
    if math.isinf(a) or math.isinf(b):
        return a == b
    return abs(a - b) <= tol * max(1.0, abs(a), abs(b))


def _check_against_highs(jm, variables=None, constraints=None):
    """Solution.variability(points=True) of jm over the oracle against HiGHS; returns the report (None: no optimum)."""
    jm = strip_timeouts(jm)
    sol = _solution(jm)
    if sol._tableau.sol.tableau is None or not (sol.feasible and sol.bounded):
        return None
    h = _Highs(jm)
    assert h.status == 0
    v = sol.variability(variables=variables, constraints=constraints, points=True)
    t = sol._tableau
    assert v["lps"] == len(t.targets) and t.batches == (1 if v["lps"] else 0)
    assert all(f.closed for f in t.faces), "the face tableau was not closed"
    if not v["exact"]:
        return v
    tol = lambda x: 1e-6 * max(1.0, abs(x))  # noqa: E731
    for vid, e in v["variables"].items():
        for side, s in (("min", -1), ("max", 1)):
            assert _close(e[side], h.variable(vid, s)), (vid, side, e, h.variable(vid, s))
            if e["arg" + side] is not None and not math.isinf(e[side]):
                h.check_point(e["arg" + side])
                assert _close(e["arg" + side][vid], e[side]), (vid, side, e)
        assert e["min"] - tol(e["value"]) <= e["value"] <= e["max"] + tol(e["value"]), (vid, e)
    for c in v["constraints"]:
        e = c["slack"]
        for side, s in (("min", -1), ("max", 1)):
            want = h.slack(c["name"], c["type"], s)
            assert _close(e[side], want), (c["name"], c["type"], side, e, want)
            if e["arg" + side] is not None and not math.isinf(e[side]):
                h.check_point(e["arg" + side])
        assert e["min"] - tol(e["value"]) <= e["value"] <= e["max"] + tol(e["value"]), (c, e)
    everything = sol.variability() if variables is not None else v
    assert v["unique"] == all(e["max"] - e["min"] <= t.precision for e in everything["variables"].values())
    return v


@pytest.mark.parametrize("fx", [f for f in CONTINUOUS if f["file"] != "Monster Problem.json"], ids=lambda f: f["file"])
def test_fixture_ranges_match_highs(fx):
    pytest.importorskip("scipy")
    if _check_against_highs(fx["model"]) is None:
        pytest.skip("no optimum")


def test_monster_problem_sampled():
    """The 600-row fixture: every 40th variable and row reported (every variable still takes part in `unique`)."""
    pytest.importorskip("scipy")
    jm = [f for f in BUNDLE["fixtures"] if f["file"] == "Monster Problem.json"][0]["model"]
    v = _check_against_highs(jm, variables=list(jm["variables"])[::40], constraints=list(jm["constraints"])[::40])
    assert v is not None and len(v["variables"]) == len(list(jm["variables"])[::40])


@pytest.mark.parametrize("seed", range(5))
def test_planted_alternative_optima_match_highs(seed):
    """alternative_optima_model: the face has dimension >= 2 (the `par` block alone gives par - 1 free columns)."""
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    v = _check_against_highs(problems.alternative_optima_model(18 + seed, 9 + seed, seed=20 + seed))
    assert v["exact"] and not v["unique"] and v["free"] >= 2 and v["lps"] > 0
    wide = [e for e in v["variables"].values() if e["max"] - e["min"] > 1e-6]
    assert len(wide) >= 2, "the planted block moves"


@pytest.mark.parametrize("seed", range(4))
def test_seeded_dense_and_mixed_lps_match_highs(seed):
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    assert _check_against_highs(problems.dense_packing_lp_model(14 + seed, 10 + seed, seed=seed)) is not None
    checked = 0
    for k in range(30):
        jm = problems.mixed_lp_model(10 + seed, 8 + seed, seed=500 + 30 * seed + k)
        v = _check_against_highs(jm)
        checked += v is not None and v["exact"]
        if checked >= 2:
            return
    pytest.fail(f"only {checked} seeded mixed LPs had an optimum")


def test_unbounded_face_has_infinite_ends():
    """max x - y, x - y <= 2: the optimal face is the ray from (2, 0) along (1, 1)."""
    pytest.importorskip("scipy")
    jm = {"optimize": "z", "opType": "max", "constraints": {"gap": {"max": 2}, "low": {"min": 1}},
          "variables": {"x": {"z": 1, "gap": 1, "low": 1}, "y": {"z": -1, "gap": -1}}}
    v = _check_against_highs(jm)
    assert v["exact"] and not v["unique"]
    assert (v["variables"]["x"]["min"], v["variables"]["x"]["max"]) == (2.0, math.inf)
    assert (v["variables"]["y"]["min"], v["variables"]["y"]["max"]) == (0.0, math.inf)
    assert v["variables"]["x"]["argmax"] is None and v["variables"]["x"]["argmin"] == {"x": 2.0, "y": 0.0}
    low = [c for c in v["constraints"] if c["name"] == "low"][0]["slack"]
    assert (low["min"], low["max"]) == (1.0, math.inf)


def test_presolve_fixed_variable():
    """-x <= -2 and x <= 2: presolve fixes x = 2; y and w share the rest of `cap` at equal cost."""
    pytest.importorskip("scipy")
    sol = _solution(FIXED)
    assert sol._tableau.model.presolveResult.fixedVariables, "presolve fixes x"
    v = _check_against_highs(FIXED)
    assert v["variables"]["x"] == dict(v["variables"]["x"], value=2, min=2, max=2, fixed=True)
    assert (v["variables"]["y"]["min"], v["variables"]["y"]["max"]) == (0.0, 5.0) and not v["unique"]
    x = [lab for lab, _ in sol._tableau.targets]
    assert all(lab != next(u for u in sol._tableau.model.variables if u.id == "x").index for lab in x)


def test_hand_example_and_berlin_airlift():
    v = _solution(HAND).variability()
    assert v["unique"] is False and v["exact"] is True
    for vid in ("x", "y"):
        assert (v["variables"][vid]["min"], v["variables"][vid]["max"], v["variables"][vid]["fixed"]) == (1.0, 3.0, False)
    slack = {c["name"]: c["slack"] for c in v["constraints"]}
    assert [c["name"] for c in v["constraints"]] == ["both", "capx", "capy"] and {c["type"] for c in v["constraints"]} == {"max"}
    assert (slack["both"]["min"], slack["both"]["max"]) == (0.0, 0.0)
    assert (slack["capx"]["min"], slack["capx"]["max"]) == (0.0, 2.0)
    b = _solution(BERLIN).variability()
    assert b["unique"] is True and b["exact"] is True
    assert (b["variables"]["brit"]["min"], b["variables"]["brit"]["max"]) == (24.0, 24.0)
    assert (b["variables"]["yank"]["min"], b["variables"]["yank"]["max"]) == (20.0, 20.0)


def test_degenerate_is_not_non_unique():
    """The Berlin Airlift fixture's vertex is primal degenerate (three rows bind at a vertex of two variables, so a
    slack is basic at 0) and its optimum is unique: no reduced cost is 0, so no LP runs.  In the second model y sits
    at reduced cost 0, so its column is kept and LPs run, but the degenerate row holds it at 0: unique all the same."""
    jm = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Berlin Air Lift Problem.json"][0]["model"])
    sol = _solution(jm)
    v = sol.variability()
    assert (sol._tableau.final_state()[0][1:] == 0).any(), "a basic variable at 0"
    assert (v["unique"], v["exact"], v["free"], v["lps"]) == (True, True, 0, 0)
    tied = {"optimize": "z", "opType": "max", "constraints": {"a": {"max": 3}, "b": {"max": 3}},
            "variables": {"x": {"z": 1, "a": 1, "b": 1}, "y": {"b": 1}}}
    w = _solution(tied).variability()
    assert w["free"] > 0 and w["lps"] > 0 and w["unique"] is True and w["exact"] is True
    assert (w["variables"]["y"]["min"], w["variables"]["y"]["max"]) == (0.0, 0.0)


def test_no_free_column_runs_no_lp():
    jm = {"optimize": "z", "opType": "max", "constraints": {"a": {"max": 4}, "b": {"max": 6}, "c": {"max": 3}},
          "variables": {"x": {"z": 3, "a": 1, "b": 1, "c": 1}, "y": {"z": 2, "a": 1, "b": 3}}}
    sol = _solution(jm)
    v = sol.variability(points=True)
    assert (v["free"], v["lps"], v["unique"], v["exact"]) == (0, 0, True, True)
    assert sol._tableau.batches == 0 and sol._tableau.faces == []
    for e in list(v["variables"].values()) + [c["slack"] for c in v["constraints"]]:
        assert e["min"] == e["value"] == e["max"]
    assert v["variables"]["x"]["argmin"] == {"x": 3.0, "y": 1.0} == v["variables"]["y"]["argmax"]


def test_rule_4_counts_and_restricted_reports():
    """Two LPs per basic label, one per non-basic label in a kept column, none for a banned column; variables= and
    constraints= restrict the report and the row targets, never the variables behind `unique`."""
    from jslpsolver_b200 import problems
    from oracle import variability as OV
    jm = problems.alternative_optima_model(20, 10, seed=3)
    sol = _solution(jm)
    t, m = sol._tableau, sol._tableau.model
    M, (vrow, vcol) = t.sol.tableau.matrix(), t.sol.tableau.maps()
    kept = set(int(c) for c in OV.face(M, vcol, 1e-8)[0])
    basic = set(int(x) for x in vrow[1:])
    col_of = {int(vcol[c]): c for c in range(1, len(vcol))}

    def lps(labels):
        return sum(2 if lab in basic else (1 if col_of[lab] in kept else 0) for lab in labels)

    v = sol.variability()
    assert v["lps"] == lps([x.index for x in m.variables] + [c.index for c in m.constraints])
    assert v["free"] == len(kept) - 1 and len(kept) < M.shape[1], "some column is banned"
    banned = [x for x in m.variables if x.index in col_of and col_of[x.index] not in kept]
    assert banned and all(v["variables"][x.id]["min"] == v["variables"][x.id]["max"] == 0.0 for x in banned)
    t.targets.clear()
    part = sol.variability(variables=["x0"], constraints=["c1"])
    assert list(part["variables"]) == ["x0"] and [c["name"] for c in part["constraints"]] == ["c1"]
    assert part["lps"] == lps([x.index for x in m.variables] + [c.index for c in m.constraints if c.name == "c1"])
    assert part["unique"] == v["unique"] and part["variables"]["x0"] == v["variables"]["x0"]
    # the oracle's own ranges say the same, label for label
    want, free, n, submitted = OV.ranges(M, vrow, vcol, 1e-8, [x.index for x in m.variables] + [c.index for c in m.constraints])
    assert (free, n) == (v["free"], v["lps"])
    for x in m.variables:
        assert (want[x.index]["min"], want[x.index]["max"]) == (v["variables"][x.id]["min"], v["variables"][x.id]["max"])
    # an equality is two rows, in tableau order
    eq = {"optimize": "z", "opType": "max", "constraints": {"mix": {"equal": 10}, "cap": {"max": 30}},
          "variables": {"x": {"z": 1, "mix": 1, "cap": 2}, "y": {"z": 1, "mix": 1, "cap": 1}}}
    se = _solution(eq)
    ve = se.variability(constraints=["mix"])
    order = [("mix", "max" if c.isUpperBound else "min") for c in se._tableau.model.constraints if c.name == "mix"]
    assert [(c["name"], c["type"]) for c in ve["constraints"]] == order and sorted(order) == [("mix", "max"), ("mix", "min")]
    assert not ve["unique"] and (ve["variables"]["x"]["min"], ve["variables"]["x"]["max"]) == (0.0, 10.0)


def test_face_rule_at_its_thresholds():
    """Rule 1 at exactly +-P, +-0, just beyond +-P and NaN; rule 2's zero row and untouched body."""
    from oracle import variability as OV
    P = 1e-8
    cost = [123.0, P, -P, 0.0, -0.0, np.nextafter(P, 1), np.nextafter(-P, -1), math.nan, 5.0, -5.0, 1e-300]
    M = np.arange(3 * len(cost), dtype=np.float64).reshape(3, len(cost)) - 7.5
    M[0] = cost
    M[2, 3] = -0.0
    kept, F, vcol_f = OV.face(M, np.arange(100, 100 + len(cost)), P)
    assert list(kept) == [0, 1, 2, 3, 4, 10] and list(vcol_f) == [100, 101, 102, 103, 104, 110]
    assert not np.signbit(F[0]).any() and (F[0] == 0).all()
    assert np.array_equal(F[1:].view(np.uint64), M[1:][:, kept].view(np.uint64))


def test_value_errors():
    from jslpsolver_b200.tableau import Solution
    sol = _solution(BERLIN)
    for kw, match in (({"variables": ["nope"]}, "no variable named"), ({"constraints": ["nope"]}, "no constraint named"),
                      ({"variables": "brit"}, "takes a list"), ({"constraints": {"plane": 1}}, "takes a list"),
                      ({"variables": 3}, "takes a list")):
        with pytest.raises(ValueError, match=r"variability\(\).*" + match):
            sol.variability(**kw)
    assert sol._tableau.batches == 0, "a refused call ran LPs"
    free = dict(BERLIN, unrestricted={"brit": 1})
    with pytest.raises(ValueError, match=r"variability\(\) does not support unrestricted variables"):
        _solution(free).variability()
    lp0 = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Berlin Air Lift Problem.json"][0]["model"])
    mip = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Integer Berlin Air Lift Problem.json"][0]["model"])
    soft = dict(lp0, constraints=dict(lp0["constraints"], plane={"max": 44, "weight": 10}))
    for model, feasible, bounded, match in ((mip, True, True, "integer or binary"), (soft, True, True, "soft constraints"),
                                            (lp0, False, True, "infeasible"), (lp0, True, False, "unbounded")):
        with pytest.raises(ValueError, match=r"variability\(\).*" + match):
            _solution(model, feasible, bounded).variability()
    s = _solution(lp0)
    s._tableau._version += 1
    with pytest.raises(ValueError, match="edited or solved again"):
        s.variability()
    s._tableau.handle = None
    with pytest.raises(ValueError, match="has not been solved"):
        Solution(s._tableau, 0.0, True, True).variability()


def test_ctypes_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+jslp_face_create\s*\(([^)]*)\)\s*;", header)
    assert proto, "jslp_face_create is not declared"
    params = [re.sub(r"\s+", " ", p.strip()) for p in proto.group(1).split(",")]
    types = [re.sub(r"\s*\b\w+$", "", p).replace(" *", "*") for p in params]
    assert types == ["jslp_tab*", "jslp_tab**", "int32_t*", "int32_t*"], types
    assert "section 2h" in header[:proto.start()][-1500:]
    (name, res, args), = [s for s in _lib.SYMBOLS if s[0] == "jslp_face_create"]
    C = _lib.C
    assert res is C.c_int and len(args) == 4 and args[0] is C.c_void_p and args[3] is C.c_void_p
    assert args[1]._type_ is C.c_void_p and args[2]._type_ is C.c_int32
    assert re.search(r"int\s+jslp_abi_version", header) and "return 2;" in open(
        os.path.join(ROOT, "jslpsolver_b200", "csrc", "jslp_api.cu")).read().split("jslp_abi_version")[1][:40]

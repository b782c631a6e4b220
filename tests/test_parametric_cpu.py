"""CPU checks of the parametric path (DESIGN.md section 2d) on optimal tableaux from the oracle: every piece against
SciPy HiGHS re-solves of the edited model, the stops just beyond the end, the monotone slopes, the first breakpoint
against the sensitivity range end, the Berlin Airlift answers, the host's name resolution and result shape over the
restatement, its ValueError cases, and the C prototype against ctypes."""
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


def _soft(jm):
    return any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())


CONTINUOUS = [f for f in BUNDLE["fixtures"] + BUNDLE["readme"]
              if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"]))
              and isinstance(f["model"].get("optimize"), str)]


def _close(a, b, tol=1e-7):
    return abs(a - b) <= tol * max(1.0, abs(a), abs(b))


def _no_presolve(jm):
    """The model as the LP the tableau holds: presolve off, so HiGHS and the tableau see the same rows and costs."""
    return dict(jm, options=dict(jm.get("options") or {}, presolve=False))


class _Lp:
    """An optimal oracle solve of jm and what the path needs from it."""

    def __init__(self, jm):
        from oracle import ref_model
        from oracle import sensitivity as S
        self.jm = jm
        self.sol = ref_model.solve_full(jm, fast_cycles=True)
        self.ok = self.sol.tableau is not None and self.sol.feasible and self.sol.bounded
        if not self.ok:
            return
        self.model = self.sol.model
        self.M = self.sol.tableau.matrix()
        self.vrow, self.vcol = self.sol.tableau.maps()
        self.unres = np.zeros(self.M.shape[0] + self.M.shape[1] - 2, dtype=np.uint8)
        for i in self.model.unrestrictedVariables:
            self.unres[i] = 1
        self.sigma = -1.0 if self.model.isMinimization else 1.0
        self.names = S.json_row_names(jm)
        self.report = S.report(jm, self.sol)

    def path(self, kind, labels, row_signs, theta0, target, cap=10000):
        from oracle import parametric as OP
        signs = OP.signs_for(kind, row_signs if kind == 0 else [self.sigma], theta0, target)
        p = OP.path(self.M, self.vrow, self.vcol, self.unres, self.model.precision, kind, labels, signs, theta0,
                    target, cap)
        return p, OP.result(p, self.sigma, theta0, target, float(self.M[0, 0]))


def _highs(jm, rows=None, cost=None):
    """linprog(HiGHS) of jm with the JSON bounds `rows` = {(name, "min"|"max"): value} and the cost `cost` = (var,
    value) replaced: ("optimal", result) / ("infeasible",) / ("unbounded",)."""
    from scipy.optimize import linprog
    names = list(jm["variables"])
    obj = jm["optimize"]
    kappa = -1.0 if jm["opType"] == "max" else 1.0
    costs = {v: jm["variables"][v].get(obj, 0.0) for v in names}
    if cost is not None:
        costs[cost[0]] = cost[1]
    c = kappa * np.array([costs[v] for v in names], dtype=np.float64)
    A, b = [], []
    for cname, spec in jm["constraints"].items():
        a = np.array([jm["variables"][v].get(cname, 0.0) for v in names], dtype=np.float64)
        lo, hi = (spec["equal"], spec["equal"]) if spec.get("equal") is not None else (spec.get("min"), spec.get("max"))
        lo = (rows or {}).get((cname, "min"), lo)
        hi = (rows or {}).get((cname, "max"), hi)
        if hi is not None:
            A.append(a); b.append(hi)
        if lo is not None:
            A.append(-a); b.append(-lo)
    free = jm.get("unrestricted") or {}
    bounds = [(None, None) if free.get(v) else (0, None) for v in names]
    res = linprog(c, A_ub=np.array(A) if A else None, b_ub=b or None, bounds=bounds, method="highs")
    if res.status == 0:
        return ("optimal", kappa * res.fun)
    assert res.status in (2, 3), res.message
    return ("infeasible",) if res.status == 2 else ("unbounded",)


def _check_path(lp, out, kind, g, evaluate, what):
    """Pieces against HiGHS, the stop just beyond the end, and monotone slopes over the pieces of non-zero length."""
    pieces = out["pieces"]
    assert pieces, what
    for k, pc in enumerate(pieces):
        assert g * (pc["to"] - pc["from"]) >= 0, (what, pc)
        if k:
            assert pc["from"] == pieces[k - 1]["to"] and pc["result"]["from"] == pieces[k - 1]["result"]["to"], what
        pts = [(pc["from"], pc["result"]["from"]), (pc["to"], pc["result"]["to"])]
        if pc["to"] != pc["from"]:
            pts.append(((pc["from"] + pc["to"]) / 2, (pc["result"]["from"] + pc["result"]["to"]) / 2))
            assert _close(pc["result"]["to"] - pc["result"]["from"], pc["slope"] * (pc["to"] - pc["from"]), 1e-7 *
                          max(1.0, abs(pc["result"]["to"]))), (what, pc)
        for theta, want in pts:
            got = evaluate(theta)
            assert got[0] == "optimal" and _close(got[1], want), (what, k, theta, got, want)
    end = out["end"]
    step = 1e-3 * max(1.0, abs(end))
    if out["stop"] == "reached":
        assert end == out["to"] if "to" in out else True
    elif out["stop"] in ("infeasible", "unbounded"):
        assert evaluate(end)[0] == "optimal", what
        assert evaluate(end + g * step)[0] == out["stop"], (what, end)
    slopes = [pc["slope"] for pc in pieces if pc["to"] != pc["from"]]
    # value function: concave in a right-hand side and convex in a cost for max, the reverse for min
    concave = (kind == 0) == (lp.sigma > 0)
    for a, b in zip(slopes, slopes[1:]):
        d = g * (b - a)  # change of d result / d theta as theta increases
        tol = 1e-9 * max(1.0, abs(a), abs(b))
        assert (d <= tol) if concave else (d >= -tol), (what, slopes)


def _targets(cur, rng_end_lo, rng_end_hi):
    out = []
    for g, end in ((1.0, rng_end_hi), (-1.0, rng_end_lo)):
        past = abs(end - cur) if math.isfinite(end) else 0.0
        out.append(cur + g * (past + 2.0 * max(1.0, abs(cur))))
    return out


def _rows_and_vars(lp, every=1):
    """(what, kind, labels, row signs, current value, evaluate(theta), first-range-end(g)) for every row, every
    equality (both rows together) and every variable that presolve did not fix."""
    jm, model = lp.jm, lp.model
    cases = []
    for k, con in enumerate(model.constraints):
        if k % every:
            continue
        name, rep = lp.names[k], lp.report["constraints"][k]
        side = "max" if con.isUpperBound else "min"
        ev = (lambda th, name=name, side=side: _highs(jm, rows={(name, side): th}))
        cases.append((f"{name}/{side}", 0, [con.index], [1.0 if con.isUpperBound else -1.0], float(con.rhs), ev,
                      rep["range"]))
    for name in {n for n in lp.names if jm["constraints"][n].get("equal") is not None}:
        rows = [c for k, c in enumerate(model.constraints) if lp.names[k] == name]
        ev = (lambda th, name=name: _highs(jm, rows={(name, "min"): th, (name, "max"): th}))
        cases.append((f"{name}/equal", 0, [c.index for c in rows], [1.0 if c.isUpperBound else -1.0 for c in rows],
                      float(rows[0].rhs), ev, None))
    for j, var in enumerate(model.variables):
        if j % every:
            continue
        ev = (lambda th, vid=var.id: _highs(jm, cost=(vid, th)))
        cases.append((f"cost {var.id}", 1, [var.index], None, float(var.cost), ev, lp.report["variables"][var.id]["range"]))
    return cases


def _run_model(jm, every=1):
    lp = _Lp(_no_presolve(jm))
    if not lp.ok:
        return 0
    n = 0
    for what, kind, labels, rs, cur, ev, rng_ in _rows_and_vars(lp, every):
        lo, hi = (rng_["min"], rng_["max"]) if rng_ else (math.inf, math.inf)
        for target in _targets(cur, lo, hi):
            g = 1.0 if target >= cur else -1.0
            p, out = lp.path(kind, labels, rs, cur, target)
            out["to"] = target
            _check_path(lp, out, kind, g, ev, f"{what} -> {target}")
            # the first breakpoint is sensitivity()'s range end, bit for bit, where that end lies on the way
            end = (hi if g > 0 else lo) if rng_ else math.inf
            if math.isfinite(end) and g * (end - cur) >= 0 and g * (target - end) > 0:
                assert p["records"][0][0] == end, (what, target, p["records"][0][0], end)
            n += 1
    return n


@pytest.mark.parametrize("fx", [f for f in CONTINUOUS if f["file"] != "Monster Problem.json"], ids=lambda f: f["file"])
def test_fixture_paths_match_highs(fx):
    """Every row, every equality and every variable of each continuous fixture, both directions, with targets past
    the sensitivity range: each piece equals HiGHS's optimum at its ends and midpoint, the stops hold just beyond the
    end, the slopes are monotone, and the first breakpoint is the range end."""
    pytest.importorskip("scipy")
    jm = strip_timeouts(fx["model"])
    lp = _Lp(_no_presolve(jm))
    if not lp.ok:
        pytest.skip("no optimum")
    assert _run_model(jm) > 0


def test_monster_problem_sampled():
    """The 600-row fixture: every 25th row and variable (the path and HiGHS both scale with the model)."""
    pytest.importorskip("scipy")
    jm = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Monster Problem.json"][0]["model"])
    assert _run_model(jm, every=25) >= 40


def _with_unrestricted(jm, every):
    jm = dict(jm)
    jm["unrestricted"] = {v: 1 for k, v in enumerate(jm["variables"]) if k % every == 0}
    return jm


@pytest.mark.parametrize("seed", range(6))
def test_seeded_mixed_lps_match_highs(seed):
    """Seeded mixed max / min LPs, half of them with unrestricted variables (the first seed of each group whose LP has
    an optimum), through the same checks."""
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    for k in range(40):
        jm = problems.mixed_lp_model(8 + seed, 6 + seed, seed=100 + 40 * seed + k)
        if seed % 2:
            jm = _with_unrestricted(jm, 4)
        for op in ("max", "min"):
            if _run_model(dict(jm, opType=op)):
                return
    pytest.fail("no seeded LP with an optimum")


def test_stops_infeasible_and_unbounded():
    """A right-hand side pushed until no point is feasible, and a cost pushed until the optimum is unbounded."""
    jm = {"optimize": "z", "opType": "max", "constraints": {"a": {"max": 10}, "b": {"min": 2}},
          "variables": {"x": {"z": 1, "a": 1, "b": 1}, "y": {"z": -1}}}
    lp = _Lp(_no_presolve(jm))
    k = lp.names.index("a")
    _, out = lp.path(0, [lp.model.constraints[k].index], [1.0], 10.0, -5.0)
    assert out["stop"] == "infeasible" and out["end"] == 2.0, out
    y = lp.model.variables[1]
    _, out = lp.path(1, [y.index], None, -1.0, 5.0)
    assert out["stop"] == "unbounded" and out["end"] == 0.0, out
    pytest.importorskip("scipy")
    assert _highs(jm, rows={("a", "max"): 1.999})[0] == "infeasible"
    assert _highs(jm, cost=("y", 0.001))[0] == "unbounded"


def test_berlin_airlift_known_answers():
    """README Berlin Airlift (max 20000 b + 30000 y; plane b + y <= 44, person 8b + 16y <= 512, cost 5000b + 9000y
    <= 300000), optimum b = 24, y = 20 (result 1 080 000) at a degenerate vertex where all three rows are tight.

    person down to 0: with y = 0 the binding rows are person and plane until 8b = 352 (b = 44): between 352 and 512
    the trade b for y along plane gives d result / d person = (30000 - 20000) / 8 = 1250, result 880 000 at 352; below
    352 only person binds, b = p / 8, slope 20000 / 8 = 2500, result 0 at p = 0.  person up to 1000: cost and plane
    already bind (5000b + 9000y = 300000, b + y = 44 gives b = 24, y = 20), so the slope is 0 and the result stays
    1 080 000.  brit cost up to 40000: b stays 24 (slope 24) until c_b / c_y = 5000 / 9000 ... the plane/cost vertex
    stops being optimal at c_b = 30000 (plane vs person: c_b = c_y = 30000 makes b = 44 on plane optimal), result
    24 * 30000 + 20 * 30000 = 1 320 000; beyond it b = 44, y = 0, slope 44, result 1 760 000 at 40000.  brit cost down
    to 10000: below c_b = 15000 (= 30000 / 2, person's ratio 8:16) the vertex b = 0, y = 32 wins, result 960 000 at
    15000 with slope 0 after it."""
    from jslpsolver_b200.tableau import Solution
    lp = _Lp(BERLIN)
    m = _cpu_model(BERLIN)
    sol = Solution(_StubTableau(m, lp), float(-lp.M[0, 0]), True, True)

    def nonzero(out):
        return [(pc["from"], pc["to"], pc["result"]["to"], pc["slope"]) for pc in out["pieces"] if pc["to"] != pc["from"]]

    out = sol.parametric(constraint="person", to=0)
    assert nonzero(out) == [(512.0, 352.0, 880000.0, 1250.0), (352.0, 0.0, 0.0, 2500.0)] and out["stop"] == "reached"
    out = sol.parametric(constraint="person", to=1000)
    assert out["pieces"][0]["to"] == 512.0 and nonzero(out) == [(512.0, 1000.0, 1080000.0, 0.0)]
    assert out["result"] == 1080000.0 and out["stop"] == "reached"
    out = sol.parametric(variable="brit", to=40000)
    assert nonzero(out) == [(20000.0, 30000.0, 1320000.0, 24.0), (30000.0, 40000.0, 1760000.0, 44.0)]
    assert out["values"] == {"brit": 44.0, "yank": 0.0}
    out = sol.parametric(variable="brit", to=10000)
    assert nonzero(out) == [(20000.0, 15000.0, 960000.0, 24.0), (15000.0, 10000.0, 960000.0, 0.0)]
    assert out["pieces"][0]["leaving"] is not None and out["pieces"][-1]["leaving"] is None


# ---------------------------------------------------------------- the host module over the restatement
class _StubTableau:
    """Stands in for GpuTableau: serves the oracle's optimal tableau and runs the restatement as the device path."""

    def __init__(self, model, lp=None):
        self.model = model
        self.handle = None
        self._version, self._solved_version = 0, -1
        self.lp = lp
        if lp is not None:
            self.handle = object()
            self._solved_version = 0
            self.height, self.width = lp.M.shape

    def final_state(self):
        return self.lp.M[:, 0].copy(), self.lp.M[0].copy(), self.lp.vrow, self.lp.vcol

    def parametric_path(self, kind, labels, signs, theta0, target, max_breaks):
        from oracle import parametric as OP
        p = OP.path(self.lp.M, self.lp.vrow, self.lp.vcol, self.lp.unres, self.lp.model.precision, kind, labels,
                    signs, theta0, target, max_breaks)
        return {"theta": [r[0] for r in p["records"]], "obj_raw": [r[1] for r in p["records"]],
                "dobj": [r[2] for r in p["records"]], "rc_lbl": [r[3:] for r in p["records"]], "stop": p["stop"],
                "end_rhs": p["end_rhs"], "end_vrow": p["end_vrow"]}


def _cpu_model(jm):
    import jslpsolver_b200.tableau as T
    from jslpsolver_b200.model import Model, presolve
    saved = T.GpuTableau
    T.GpuTableau = lambda *a, **k: None
    try:
        m = Model().loadJson(jm)
    finally:
        T.GpuTableau = saved
    m.presolveResult = presolve(m)
    for v in m.presolveResult.fixedVariables:
        v.cost = 0
    return m


@pytest.mark.parametrize("fx", [f for f in CONTINUOUS if f["file"] != "Monster Problem.json"], ids=lambda f: f["file"])
def test_host_result_matches_the_restatement(fx):
    """Solution.parametric()'s host side (name resolution, signs, equalities, labels to names, values) over the
    restatement equals the restatement's own pieces for every row name and variable, both directions."""
    from jslpsolver_b200.tableau import Solution
    jm = strip_timeouts(fx["model"])
    lp = _Lp(jm)
    if not lp.ok:
        pytest.skip("no optimum")
    m = _cpu_model(jm)
    sol = Solution(_StubTableau(m, lp), 0.0, True, True)
    fixed = m.presolveResult.fixedVariables
    for name in dict.fromkeys(lp.names):
        spec = jm["constraints"][name]
        sides = [None] if spec.get("equal") is not None or len([k for k in ("min", "max") if spec.get(k) is not None]) == 1 \
            else ["min", "max"]
        for side in sides:
            rows = [c for k, c in enumerate(m.constraints) if lp.names[k] == name and (side is None or c.isUpperBound == (side == "max"))]
            cur = float(rows[0].rhs)
            for target in (cur + 7.0 * max(1.0, abs(cur)), cur - 7.0 * max(1.0, abs(cur))):
                got = sol.parametric(constraint=name, side=side, to=target)
                _, want = lp.path(0, [c.index for c in rows], [1.0 if c.isUpperBound else -1.0 for c in rows], cur, target)
                _same(got, want, lp, m)
                assert got["kind"] == "rhs" and got["name"] == name and got["from"] == cur and got["to"] == target
                assert got["side"] == (side or ("equal" if len(rows) == 2 else ("max" if rows[0].isUpperBound else "min")))
    for v in m.variables:
        if v in fixed:
            with pytest.raises(ValueError, match="presolve fixed"):
                sol.parametric(variable=v.id, to=1.0)
            continue
        for target in (v.cost + 5.0 * max(1.0, abs(v.cost)), v.cost - 5.0 * max(1.0, abs(v.cost))):
            got = sol.parametric(variable=v.id, to=target)
            _, want = lp.path(1, [v.index], None, float(v.cost), target)
            _same(got, want, lp, m)
            assert got["kind"] == "cost" and got["side"] is None


def _same(got, want, lp, m):
    by_index = {c.index: c for c in m.constraints}
    var_of = {v.index: v.id for v in m.variables}

    def ref(label):
        if label is None:
            return None
        if label in var_of:
            return {"variable": var_of[label]}
        c = by_index[label]
        return {"constraint": c.name if c.name is not None else c.index, "type": "max" if c.isUpperBound else "min"}

    assert got["stop"] == want["stop"] and got["end"] == want["end"] and got["result"] == want["result"]
    assert len(got["pieces"]) == len(want["pieces"])
    for a, b in zip(got["pieces"], want["pieces"]):
        assert a == dict(b, leaving=ref(b["leaving"]), entering=ref(b["entering"]))


def test_value_errors():
    """Unknown names, a min+max constraint without side, both or neither of constraint / variable, a bad target, a
    presolve-fixed variable, and every case sensitivity() refuses."""
    from jslpsolver_b200 import parametric as HP
    from jslpsolver_b200.tableau import Solution
    jm = dict(BERLIN, constraints=dict(BERLIN["constraints"], labor={"min": 1, "max": 50}),
              variables={k: dict(v, labor=1) for k, v in BERLIN["variables"].items()})
    lp = _Lp(jm)
    m = _cpu_model(jm)
    sol = Solution(_StubTableau(m, lp), 0.0, True, True)
    for kw, match in ((dict(constraint="nope", to=1), "no constraint named"), (dict(variable="nope", to=1), "no variable named"),
                      (dict(constraint="labor", to=1), "pass side"), (dict(constraint="person", side="min", to=1), "only a 'max'"),
                      (dict(constraint="labor", side="equal", to=1), "not an equality"),
                      (dict(constraint="person", variable="brit", to=1), "exactly one"), (dict(to=1), "exactly one"),
                      (dict(constraint="person", to=None), "finite target"), (dict(constraint="person", to=math.inf), "finite target"),
                      (dict(variable="brit", side="max", to=1), "constraints only")):
        with pytest.raises(ValueError, match=match):
            sol.parametric(**kw)
    assert sol.parametric(constraint="labor", side="max", to=60)["side"] == "max"
    out = HP.compute(sol, constraint="person", to=0, max_breaks=1)
    assert out["stop"] == "limit" and len(out["pieces"]) == 1 and out["pieces"][0]["leaving"] is not None
    # the cases sensitivity() refuses, with parametric() named in the message
    lp0 = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Berlin Air Lift Problem.json"][0]["model"])
    mip = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Integer Berlin Air Lift Problem.json"][0]["model"])
    soft = dict(lp0, constraints=dict(lp0["constraints"], plane={"max": 44, "weight": 10}))
    for model, feasible, bounded, match in ((mip, True, True, "integer or binary"), (soft, True, True, "soft constraints"),
                                            (lp0, False, True, "infeasible"), (lp0, True, False, "unbounded"),
                                            (lp0, True, True, "has not been solved")):
        with pytest.raises(ValueError, match=r"parametric\(\).*" + match):
            Solution(_StubTableau(_cpu_model(model)), 0.0, feasible, bounded).parametric(constraint="plane", to=1)
    t = _StubTableau(m, lp)
    s = Solution(t, 0.0, True, True)
    t._version += 1
    with pytest.raises(ValueError, match="edited or solved again"):
        s.parametric(constraint="person", to=1)
    fixed = {"optimize": "z", "opType": "max", "constraints": {"one": {"max": 0}, "cap": {"max": 5}},
             "variables": {"x": {"z": 1, "one": 1, "cap": 1}, "y": {"z": 2, "cap": 1}}}
    mf = _cpu_model(fixed)
    if mf.presolveResult.fixedVariables:
        lpf = _Lp(fixed)
        with pytest.raises(ValueError, match="presolve fixed"):
            Solution(_StubTableau(mf, lpf), 0.0, True, True).parametric(variable="x", to=3)


def test_ctypes_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+jslp_parametric\s*\(([^)]*)\)\s*;", header)
    assert proto, "jslp_parametric is not declared"
    params = [re.sub(r"\s+", " ", p.strip()) for p in proto.group(1).split(",")]
    types = [re.sub(r"\s*\b\w+$", "", p).replace(" *", "*") for p in params]
    want = ["jslp_tab*", "int", "const int32_t*", "const double*", "int", "double", "double", "int", "double*",
            "double*", "double*", "int32_t*", "int*", "int*", "double*", "int32_t*"]
    assert types == want, types
    (name, res, args), = [s for s in _lib.SYMBOLS if s[0] == "jslp_parametric"]
    C = _lib.C
    ctype = {"int": C.c_int, "double": C.c_double}
    assert res is C.c_int and len(args) == len(want)
    for a, w in zip(args, want):
        if w.endswith("*"):
            assert a is C.c_void_p or (w == "int*" and a._type_ is C.c_int), (w, a)
        else:
            assert a is ctype[w], (w, a)

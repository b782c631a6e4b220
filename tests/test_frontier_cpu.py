"""CPU checks of the two-objective frontier (DESIGN.md section 2g) over oracle/frontier.py: the Berlin Airlift answer
derived by hand, every vertex and every edge midpoint efficient by SciPy HiGHS, HiGHS's weighted optimum in the middle
of each weight interval, the lexicographic ends, unbounded stops, aligned objectives, the ends against
MultiObjective, the pricing formula against the final cost row, the host's result shaping over the restatement, the
refusals and the C prototype."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_bundle
from helpers import strip_timeouts

BUNDLE = load_bundle()
BERLIN = {"optimize": {"capacity": "max", "cost": "min"},
          "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
          "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                        "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}


def _soft(jm):
    return any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())


CONTINUOUS = [f for f in BUNDLE["fixtures"] + BUNDLE["readme"]
              if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"]))
              and isinstance(f["model"].get("optimize"), str) and f["file"] != "Monster Problem.json"]


def _close(a, b, tol=1e-7):
    return abs(a - b) <= tol * max(1.0, abs(a), abs(b))


def _with_second(jm, sense, seed, lo=0, hi=20):
    """jm with a seeded second objective `second_obj` of the given sense after its own objective."""
    rng = np.random.default_rng(seed)
    jm = strip_timeouts(jm)
    for v in jm["variables"].values():
        v["second_obj"] = float(rng.integers(lo, hi + 1))
    return dict(jm, optimize={jm["optimize"]: "max" if jm.get("opType") == "max" else "min", "second_obj": sense})


class _Lp:
    """HiGHS over the JSON model: A_ub x <= b_ub, bounds, and the sense-applied objective vectors g1, g2."""

    def __init__(self, jm):
        names = list(jm["variables"])
        self.names = names
        keys = list(jm["optimize"])
        self.g = [np.array([(1.0 if jm["optimize"][k] == "max" else -1.0) * float(jm["variables"][v].get(k) or 0.0)
                            for v in names]) for k in keys]
        A, b = [], []
        for cname, spec in jm["constraints"].items():
            a = np.array([float(jm["variables"][v].get(cname) or 0.0) for v in names])
            lo, hi = (spec["equal"], spec["equal"]) if spec.get("equal") is not None else (spec.get("min"), spec.get("max"))
            if hi is not None:
                A.append(a); b.append(hi)
            if lo is not None:
                A.append(-a); b.append(-lo)
        free = jm.get("unrestricted") or {}
        self.bounds = [(None, None) if free.get(v) else (0, None) for v in names]
        self.A, self.b = np.array(A).reshape(len(A), len(names)), np.array(b, dtype=np.float64)

    def maximise(self, c, extra=()):
        """max c.x over the model plus rows (a, b) meaning a.x >= b: ("optimal", value, x) or (status,)."""
        from scipy.optimize import linprog
        A, b = list(self.A), list(self.b)
        for a, rhs in extra:
            A.append(-np.asarray(a)); b.append(-rhs)
        res = linprog(-np.asarray(c), A_ub=np.array(A) if A else None, b_ub=b or None, bounds=self.bounds, method="highs")
        if res.status == 0:
            return ("optimal", -res.fun, res.x)
        assert res.status in (2, 3), res.message
        return ("infeasible",) if res.status == 2 else ("unbounded",)


def check_frontier(jm, what):
    """The frontier of jm over the oracle against HiGHS.  Returns the result (None when the first objective is
    unbounded)."""
    from oracle import frontier as OF
    lp = _Lp(jm)
    try:
        res, _ = OF.Frontier(jm)
    except ValueError:
        assert lp.maximise(lp.g[0])[0] == "unbounded", what
        return None
    if not res["feasible"]:
        if not jm.get("unrestricted"):  # the reference's verdicts with unrestricted variables can differ from HiGHS's
            assert lp.maximise(lp.g[0])[0] == "infeasible", what
        return res
    keys = list(jm["optimize"])
    sig = [1.0 if jm["optimize"][k] == "max" else -1.0 for k in keys]
    verts = res["vertices"]
    assert verts, what
    # tolerances relative to the largest objective value on the frontier: one objective can move by a large multiple
    # of the other's slack
    S = max(abs(v["objectives"][k]) for v in verts for k in keys)

    def near(x, y):
        return abs(x - y) <= 1e-7 * max(1.0, abs(x), abs(y), S)

    def _slack(x):
        return 1e-13 * max(1.0, abs(x))

    gv = []
    for k, v in enumerate(verts):
        x = np.array([v["values"][n] for n in lp.names])
        g1, g2 = sig[0] * v["objectives"][keys[0]], sig[1] * v["objectives"][keys[1]]
        assert near(g1, float(lp.g[0] @ x)) and near(g2, float(lp.g[1] @ x)), (what, v)
        gv.append((g1, g2, x))
        # efficient: neither objective can improve without the other getting worse (where an unbounded edge starts,
        # the second objective may also grow without bound while the first stays)
        got = lp.maximise(lp.g[1], [(lp.g[0], g1 - _slack(g1))])
        ray = res["stop"] == "unbounded" and k == len(verts) - 1 and got[0] == "unbounded"
        assert ray or (got[0] == "optimal" and near(got[1], g2)), (what, "max g2 | g1", v, got[:2])
        got = lp.maximise(lp.g[0], [(lp.g[1], g2 - _slack(g2))])
        assert got[0] == "optimal" and near(got[1], g1), (what, "max g1 | g2", v, got[:2])
        lo, hi = v["weight"]["from"], v["weight"]["to"]
        assert 0.0 <= lo <= hi <= 1.0, (what, v)
        if hi > lo:  # the weighted optimum in the middle of the interval is this vertex's weighted value
            w = (lo + hi) / 2
            got = lp.maximise((1 - w) * lp.g[0] + w * lp.g[1])
            assert got[0] == "optimal" and near(got[1], (1 - w) * g1 + w * g2), (what, "weighted", w, got[:2])
    for k in range(1, len(verts)):
        assert verts[k]["weight"]["from"] == verts[k - 1]["weight"]["to"], what
    for (a1, a2, xa), (b1, b2, xb) in zip(gv, gv[1:]):  # edge midpoints are efficient: no vertex is missing
        m1, m2 = (a1 + b1) / 2, (a2 + b2) / 2
        got = lp.maximise(lp.g[1], [(lp.g[0], m1 - _slack(m1))])
        assert got[0] == "optimal" and near(got[1], m2), (what, "midpoint", got[:2], m2)
    assert verts[0]["weight"]["from"] == 0.0, what
    # the first end: the lexicographic optimum (first objective, then second)
    b1 = lp.maximise(lp.g[0])
    lex = lp.maximise(lp.g[1], [(lp.g[0], b1[1] - _slack(b1[1]))])
    assert near(gv[0][0], b1[1]), (what, "first end")
    assert (lex[0] == "unbounded" and res["stop"] == "unbounded") or near(gv[0][1], lex[1]), (what, "first end")
    if res["stop"] == "reached":
        assert res["end"] == 1.0 and verts[-1]["weight"]["to"] == 1.0, what
        b2 = lp.maximise(lp.g[1])
        lex = lp.maximise(lp.g[0], [(lp.g[1], b2[1] - _slack(b2[1]))])
        assert near(gv[-1][1], b2[1]) and near(gv[-1][0], lex[1]), (what, "second end")
    else:
        assert res["stop"] == "unbounded", (what, res["stop"])
        # within the precision of weight 1 an unbounded stop can come from rounding (DESIGN.md section 7)
        if 1 - res["end"] > 1e-8:
            w = res["end"] + 1e-3 * (1 - res["end"])
            assert lp.maximise((1 - w) * lp.g[0] + w * lp.g[1])[0] == "unbounded", (what, res["end"])
    return res


@pytest.mark.parametrize("sense", ["max", "min"])
@pytest.mark.parametrize("fx", CONTINUOUS, ids=lambda f: f["file"])
def test_fixture_frontiers_match_highs(fx, sense):
    pytest.importorskip("scipy")
    check_frontier(_with_second(fx["model"], sense, 11), f"{fx['file']} {sense}")


@pytest.mark.parametrize("seed", range(4))
def test_dense_packing_multi_models_match_highs(seed):
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    jm = problems.dense_packing_multi_model(10 + 3 * seed, 8 + 2 * seed, 2, seed)
    for second in ("max", "min"):
        res = check_frontier(dict(jm, optimize={"profit": "max", "attr1": second}), f"dense {seed} {second}")
        assert res["stop"] == "reached"


def _mixed(seed, equal=False, free=False):
    from jslpsolver_b200 import problems
    jm = problems.mixed_lp_model(9 + seed, 6 + seed, seed=300 + seed)
    rng = np.random.default_rng(seed)
    for v in jm["variables"].values():
        v["second"] = float(rng.integers(-5, 20))
    if equal:
        name = next(k for k, s in jm["constraints"].items() if "max" in s)
        jm["constraints"][name] = {"equal": jm["constraints"][name]["max"] / 4}
    if free:
        jm["unrestricted"] = {v: 1 for k, v in enumerate(jm["variables"]) if k % 4 == 0}
    return dict(jm, optimize={"objective": jm["opType"], "second": "min" if seed % 2 else "max"})


@pytest.mark.parametrize("equal,free", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("seed", range(4))
def test_mixed_lps_match_highs(seed, equal, free):
    pytest.importorskip("scipy")
    check_frontier(_mixed(seed, equal, free), f"mixed {seed} equal={equal} free={free}")


def test_presolve_fixed_variable():
    """A variable fixed by presolve (x = 2 by a min and a max row) takes its value and adds to both objectives."""
    pytest.importorskip("scipy")
    jm = {"optimize": {"a": "max", "b": "max"},
          "constraints": {"fx": {"min": 2, "max": 2}, "cap": {"max": 10}, "mix": {"max": 12}},
          "variables": {"x": {"fx": 1, "a": 3, "b": 1}, "y": {"cap": 1, "mix": 1, "a": 2, "b": 1},
                        "z": {"cap": 1, "mix": 3, "a": 1, "b": 4}}}
    res = check_frontier(jm, "fixed")
    assert all(v["values"]["x"] == 2 for v in res["vertices"]) and len(res["vertices"]) >= 2


def test_berlin_airlift_known_answer():
    """max capacity 20000 b + 30000 y against min cost 5000 b + 9000 y (plane b + y <= 44, person 8b + 16y <= 512,
    cost <= 300000).  b = 24, y = 20 (1 080 000 / 300 000) while (1 - w) * 10000 >= w * 4000 on the trade of y for b
    along plane and cost (10000 capacity for 4000 cost): w <= 5/7.  Then b = 44 (880 000 / 220 000) while
    (1 - w) * 20000 >= w * 5000 on b alone: w <= 4/5.  Then the origin."""
    from oracle import frontier as OF
    res, _ = OF.Frontier(BERLIN)
    assert res["stop"] == "reached" and res["end"] == 1.0 and res["objectives"] == {"capacity": "max", "cost": "min"}
    want = [({"brit": 24, "yank": 20}, 1080000, 300000, 0.0, 5 / 7), ({"brit": 44, "yank": 0}, 880000, 220000, 5 / 7, 4 / 5),
            ({"brit": 0, "yank": 0}, 0, 0, 4 / 5, 1.0)]
    assert len(res["vertices"]) == 3
    for v, (vals, cap, cost, lo, hi) in zip(res["vertices"], want):
        assert all(abs(v["values"][k] - x) <= 1e-12 for k, x in vals.items()), v
        assert _close(v["objectives"]["capacity"], cap, 1e-12) and _close(v["objectives"]["cost"], cost, 1e-12), v
        assert abs(v["weight"]["from"] - lo) <= 1e-12 and abs(v["weight"]["to"] - hi) <= 1e-12, v


def test_unbounded_second_objective_and_aligned_objectives():
    pytest.importorskip("scipy")
    jm = {"optimize": {"z": "max", "w": "max"}, "constraints": {"a": {"max": 10}, "b": {"max": 4}},
          "variables": {"x": {"z": 1, "w": 1, "a": 1}, "y": {"z": 0, "w": 1, "b": -1}}}
    res = check_frontier(jm, "unbounded second")
    assert res["stop"] == "unbounded" and res["vertices"][-1]["values"] == {"x": 10.0, "y": 0.0}
    aligned = dict(jm, optimize={"z": "max", "z2": "max"},
                   variables={"x": {"z": 1, "z2": 2, "a": 1}, "y": {"z": 3, "z2": 6, "a": 1, "b": 1}})
    res = check_frontier(aligned, "aligned")
    assert len(res["vertices"]) == 1 and res["vertices"][0]["weight"] == {"from": 0.0, "to": 1.0}


class _OracleSolver:
    def Solve(self, model, precision=None, full=False, validate=False):
        from jslpsolver_b200 import validation
        from oracle import ref_model
        return ref_model.Solve(validation.validate(model) if validate else model, precision)


@pytest.mark.parametrize("seed", range(3))
def test_ends_equal_multiobjective_vertices(seed):
    """Where each single-objective optimum is unique, the first and last vertices are MultiObjective's vertices."""
    from jslpsolver_b200.polyopt import Polyopt
    from jslpsolver_b200 import problems
    from oracle import frontier as OF
    jm = problems.dense_packing_multi_model(9 + seed, 7 + seed, 2, 40 + seed)
    res, _ = OF.Frontier(jm)
    po = Polyopt(_OracleSolver(), jm)
    ends = [res["vertices"][0]["values"], res["vertices"][-1]["values"]]
    assert len(po["vertices"]) == 2
    for got, want in zip(ends, po["vertices"]):
        for k, x in got.items():
            # Solve() rounds its values to the precision (1e-8): the vertices agree to that rounding
            assert abs(x - want.get(k, 0)) <= 0.5e-8 + 1e-9 * abs(x), (k, x, want.get(k))


@pytest.mark.parametrize("fx", CONTINUOUS, ids=lambda f: f["file"])
def test_pricing_formula_reproduces_the_final_cost_row(fx):
    """R1 by the contract's pricing with C1 (the first objective's own row-0 entries) is the final row 0 to 1e-9."""
    from oracle import frontier as OF
    from oracle import ref_model
    sol = ref_model.solve_full(strip_timeouts(fx["model"]))
    if sol.tableau is None or not (sol.feasible and sol.bounded):
        pytest.skip("no optimum")
    m = sol.model
    M = sol.tableau.matrix()
    vrow, vcol = sol.tableau.maps()
    sign = -1.0 if m.isMinimization else 1.0
    c1 = np.zeros(len(m.variables) + len(m.constraints))
    for v in m.variables:
        c1[v.index] = sign * v.cost
    R1, E = OF.price(M, vrow, vcol, c1)
    scale = max(1.0, float(np.abs(M[0]).max()))
    assert np.all(np.abs(R1 - M[0]) <= 1e-9 * scale), (R1, M[0])
    assert np.all(np.abs(E) <= 1e-9 * scale)


@pytest.mark.parametrize("name", ["berlin", "dense", "mixed", "fixed"])
def test_host_result_matches_the_restatement(name):
    """frontier.result() (the host's shaping) over the restatement's path output equals the oracle's Frontier()."""
    from jslpsolver_b200 import frontier as HF
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model, presolve
    from oracle import frontier as OF
    import jslpsolver_b200.tableau as T
    jm = {"berlin": BERLIN, "dense": problems.dense_packing_multi_model(12, 9, 2, 3), "mixed": _mixed(0, True, True),
          "fixed": {"optimize": {"a": "max", "b": "min"},
                    "constraints": {"fx": {"equal": 2}, "cap": {"max": 10}},
                    "variables": {"x": {"fx": 1, "a": 3, "b": 1}, "y": {"cap": 1, "a": 2, "b": 1}}}}[name]
    want, det = OF.Frontier(jm)
    keys, senses = HF._objectives(jm)
    working = dict(jm, optimize=keys[0], opType=senses[keys[0]])
    saved = T.GpuTableau
    T.GpuTableau = lambda *a, **k: None
    try:
        m = Model().loadJson(working)
    finally:
        T.GpuTableau = saved
    m.presolveResult = presolve(m)
    for v in m.presolveResult.fixedVariables:
        v.cost = 0
    c2 = HF.cost_row(m, working, keys[1], senses[keys[1]], len(m.variables) + len(m.constraints))
    assert np.array_equal(np.array(c2).view(np.uint64), det["c2"].view(np.uint64))
    p = det["path"]
    out = {"theta": [r[0] for r in p["records"]], "rc_lbl": [r[3:] for r in p["records"]], "stop": p["stop"],
           "pt_rhs": [x[0] for x in p["points"]], "pt_vrow": [x[1] for x in p["points"]],
           "pt_break": [x[2] for x in p["points"]]}
    assert HF.result(m, working, keys, senses, out) == want


class _StubSolver:
    """Serves a solution with the given verdict; Frontier must refuse before it solves anything else."""

    def __init__(self, feasible=True, bounded=True):
        self.verdict = (feasible, bounded)

    def _instance(self, model, precision):
        verdict = self.verdict

        class _Inst:
            def solve(self):
                class _Sol:
                    feasible, bounded = verdict
                return _Sol()
        return _Inst()


def test_refusals():
    from jslpsolver_b200.frontier import Frontier
    s = _StubSolver()
    one = dict(BERLIN, optimize={"capacity": "max"})
    three = dict(BERLIN, optimize={"capacity": "max", "cost": "min", "plane": "max"})
    for model, match in ((one, "exactly two"), (three, "exactly two"), (dict(BERLIN, optimize="capacity"), "exactly two"),
                         (dict(BERLIN, ints={"brit": 1}), "integer or binary"),
                         (dict(BERLIN, binaries={"yank": 1}), "integer or binary"),
                         (dict(BERLIN, constraints=dict(BERLIN["constraints"], plane={"max": 44, "weight": 3})), "soft"),
                         (dict(BERLIN, constraints=dict(BERLIN["constraints"], plane={"max": 44, "priority": "strong"})),
                          "soft")):
        with pytest.raises(ValueError, match=match):
            Frontier(s, model)
    with pytest.raises(NotImplementedError):
        Frontier(s, dict(BERLIN, external={"solver": "x"}))
    with pytest.raises(ValueError, match="other way round"):
        Frontier(_StubSolver(bounded=False), BERLIN)
    res = Frontier(_StubSolver(feasible=False), BERLIN)
    assert res["feasible"] is False and res["vertices"] == [] and res["pivots"] == 0


def test_ctypes_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+jslp_frontier\s*\(([^)]*)\)\s*;", header)
    assert proto, "jslp_frontier is not declared"
    params = [re.sub(r"\s+", " ", p.strip()) for p in proto.group(1).split(",")]
    types = [re.sub(r"\s*\b\w+$", "", p).replace(" *", "*") for p in params]
    want = ["jslp_tab*", "const double*", "int", "int", "double*", "double*", "double*", "double*", "double*",
            "int32_t*", "int*", "int*", "double*", "int32_t*", "int32_t*", "int*", "double*", "int32_t*"]
    assert types == want, types
    (name, res, args), = [s for s in _lib.SYMBOLS if s[0] == "jslp_frontier"]
    C = _lib.C
    ctype = {"int": C.c_int, "double": C.c_double}
    assert res is C.c_int and len(args) == len(want)
    for a, w in zip(args, want):
        if w.endswith("*"):
            assert a is C.c_void_p or (w == "int*" and a._type_ is C.c_int), (w, a)
        else:
            assert a is ctype[w], (w, a)

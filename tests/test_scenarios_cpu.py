"""CPU checks of what-if scenarios (DESIGN.md section 2e): the oracle definition against SciPy HiGHS solving each edited
model from scratch, the host's edit list against the literal Model-API path (a recording tableau), Solution.scenarios()
shaped over the oracle definition, the Berlin Airlift answers, every ValueError, and the C prototype and edit struct
against the header."""
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


def _no_presolve(jm):
    return dict(jm, options=dict(jm.get("options") or {}, presolve=False))


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


def _edited_json(jm, spec):
    """jm with the spec's right-hand sides and costs written into the JSON model."""
    jm = dict(jm, constraints={k: dict(v) for k, v in jm["constraints"].items()},
              variables={k: dict(v) for k, v in jm["variables"].items()})
    for name, value in (spec.get("rhs") or {}).items():
        c = jm["constraints"][name]
        if isinstance(value, dict):
            c.update(value)
        elif c.get("equal") is not None:
            c["equal"] = value
        elif c.get("min") is not None and c.get("max") is not None:
            c["min"] = c["max"] = value
        else:
            c["max" if c.get("max") is not None else "min"] = value
    for vid, value in (spec.get("cost") or {}).items():
        jm["variables"][vid][jm["optimize"]] = value
    return jm


def _highs(jm):
    """linprog(HiGHS) of the JSON LP: ("optimal", result) / ("infeasible",) / ("unbounded",)."""
    from scipy.optimize import linprog
    names = list(jm["variables"])
    obj = jm["optimize"]
    kappa = -1.0 if jm.get("opType") == "max" else 1.0
    c = kappa * np.array([jm["variables"][v].get(obj, 0.0) for v in names], dtype=np.float64)
    A, b = [], []
    for cname, spec in jm["constraints"].items():
        a = np.array([jm["variables"][v].get(cname, 0.0) for v in names], dtype=np.float64)
        lo, hi = (spec["equal"], spec["equal"]) if spec.get("equal") is not None else (spec.get("min"), spec.get("max"))
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


def _close(a, b, tol=1e-7):
    return abs(a - b) <= tol * max(1.0, abs(a), abs(b))


def _perturbations(jm, m, sol, n, seed, every=1):
    """n seeded specs: +-10 % on the right-hand sides of about a third of the named rows and on the costs of about a
    third of the variables (every `every`-th name taking part)."""
    rng = np.random.default_rng(seed)
    names = list(jm["constraints"])[::every]
    vids = [v.id for v in m.variables][::every]
    specs = []
    for _ in range(n):
        spec = {"rhs": {}, "cost": {}}
        for name in names:
            if rng.random() > 0.35:
                continue
            c = jm["constraints"][name]
            f = lambda x: float(x) * (1.0 + rng.uniform(-0.1, 0.1)) + rng.uniform(-0.5, 0.5)  # noqa: E731
            if c.get("equal") is not None or c.get("min") is None or c.get("max") is None:
                spec["rhs"][name] = f(c.get("equal", c.get("max", c.get("min"))))
            else:
                spec["rhs"][name] = {"min": f(c["min"]), "max": f(c["max"])}
        for vid in vids:
            if rng.random() < 0.35:
                spec["cost"][vid] = float(jm["variables"][vid].get(jm["optimize"], 0.0)) * (1.0 + rng.uniform(-0.1, 0.1))
        specs.append(spec)
    return specs


def _check_against_highs(jm, specs):
    """The oracle definition of each spec against HiGHS on the edited JSON model; returns the scenarios checked."""
    from jslpsolver_b200.scenarios import edits_of
    from oracle import ref_model
    from oracle import scenarios as OS
    jm = _no_presolve(jm)
    sol = ref_model.solve_full(jm, fast_cycles=True)
    if sol.tableau is None or not (sol.feasible and sol.bounded):
        return 0
    m = _cpu_model(jm)
    n = 0
    for spec in specs:
        edits = edits_of(m, spec)
        st, _ = OS.run(sol, edits)
        if st.cyclePhase:  # the cycle check declares the scenario infeasible: HiGHS has no counterpart
            continue
        got = OS.result(sol, edits)
        want = _highs(_edited_json(jm, spec))
        verdict = "infeasible" if not got["feasible"] else ("unbounded" if not got["bounded"] else "optimal")
        assert verdict == want[0], (spec, got, want)
        if verdict == "optimal":
            assert _close(got["result"], want[1]), (spec, got["result"], want[1])
        n += 1
    return n


@pytest.mark.parametrize("fx", [f for f in CONTINUOUS if f["file"] != "Monster Problem.json"], ids=lambda f: f["file"])
def test_fixture_scenarios_match_highs(fx):
    pytest.importorskip("scipy")
    jm = strip_timeouts(fx["model"])
    from oracle import ref_model
    sol = ref_model.solve_full(_no_presolve(jm), fast_cycles=True)
    if sol.tableau is None or not (sol.feasible and sol.bounded):
        pytest.skip("no optimum")
    specs = _perturbations(jm, _cpu_model(_no_presolve(jm)), sol, 12, seed=len(fx["file"]))
    assert _check_against_highs(jm, specs) > 0


def test_monster_problem_sampled():
    """The 600-row fixture: a few scenarios over every 25th row and variable."""
    pytest.importorskip("scipy")
    jm = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Monster Problem.json"][0]["model"])
    from oracle import ref_model
    sol = ref_model.solve_full(_no_presolve(jm), fast_cycles=True)
    specs = _perturbations(jm, _cpu_model(_no_presolve(jm)), sol, 3, seed=7, every=25)
    assert _check_against_highs(jm, specs) >= 2


def _with_unrestricted(jm, every):
    jm = dict(jm)
    jm["unrestricted"] = {v: 1 for k, v in enumerate(jm["variables"]) if k % every == 0}
    return jm


@pytest.mark.parametrize("seed", range(6))
def test_seeded_mixed_lps_match_highs(seed):
    """Seeded mixed LPs (min and max rows), odd seeds with unrestricted variables, until 8 scenarios are checked.  (A
    re-solve from an optimum where an unrestricted basic variable is negative starts with phase-1 pivots and often
    cycles, which declares the scenario infeasible: those scenarios have no HiGHS counterpart and are not counted.)"""
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    from oracle import ref_model
    checked = 0
    for k in range(40):
        jm = problems.mixed_lp_model(10 + seed, 8 + seed, seed=300 + 40 * seed + k)
        if seed % 2:
            jm = _with_unrestricted(jm, 6)
        for op in ("max", "min"):
            jm = dict(jm, opType=op)
            sol = ref_model.solve_full(_no_presolve(jm), fast_cycles=True)
            if sol.tableau is None or not (sol.feasible and sol.bounded):
                continue
            specs = _perturbations(jm, _cpu_model(_no_presolve(jm)), sol, 10, seed=seed)
            checked += _check_against_highs(jm, specs)
            if checked >= 8:
                return
    pytest.fail(f"only {checked} scenarios of seeded LPs checked")


EQ_MINMAX = {"optimize": "z", "opType": "max",
             "constraints": {"mix": {"equal": 10}, "band": {"min": 2, "max": 8}, "cap": {"max": 30}},
             "variables": {"x": {"z": 3, "mix": 1, "band": 1, "cap": 2}, "y": {"z": 2, "mix": 1, "cap": 1},
                           "w": {"z": 1, "band": 1, "cap": 1}}}


def test_equal_and_min_max_constraints_match_highs():
    pytest.importorskip("scipy")
    specs = [{"rhs": {"mix": 12}}, {"rhs": {"mix": 4, "band": {"min": 3}}}, {"rhs": {"band": {"max": 5, "min": 1}}},
             {"rhs": {"band": {"min": 6, "max": 6}}, "cost": {"w": 9}}, {"rhs": {"mix": 0}, "cost": {"x": -1}},
             {"rhs": {"band": {"min": 9}}}, {"rhs": {"mix": 40}}]
    assert _check_against_highs(EQ_MINMAX, specs) == len(specs)
    assert _check_against_highs(dict(EQ_MINMAX, opType="min"), specs) == len(specs)


def test_infeasible_and_unbounded_scenarios():
    """A right-hand side that leaves no feasible point and a cost that makes the optimum unbounded, as HiGHS sees
    them; the infeasible one keeps the solved result (finish_lp_flags leaves the evaluation), the unbounded one reports
    +inf for a max model."""
    pytest.importorskip("scipy")
    jm = {"optimize": "z", "opType": "max", "constraints": {"a": {"max": 10}, "b": {"min": 2}},
          "variables": {"x": {"z": 1, "a": 1, "b": 1}, "y": {"z": -1}}}
    specs = [{"rhs": {"a": 1.5}}, {"cost": {"y": 0.5}}, {"rhs": {"a": 1.5}, "cost": {"y": 0.5}}]
    assert _check_against_highs(jm, specs) == 3
    sol = _solution(jm)
    inf, unb, both = sol.scenarios(specs)
    assert (inf["feasible"], inf["result"], inf["bounded"]) == (False, 10.0, True), inf
    assert (unb["feasible"], unb["result"], unb["bounded"]) == (True, math.inf, False), unb
    assert both["feasible"] is False


# ---------------------------------------------------------------- the host's edit list and Solution.scenarios()
class _Recorder:
    """A tableau that records what the Model API passes to it."""

    def __init__(self):
        self.calls = []

    def updateRightHandSide(self, constraint, difference):
        self.calls.append((0, constraint.index, float(difference)))

    def updateCost(self, variable, difference):
        self.calls.append((1, variable.index, float(difference)))


def _literal(jm, spec):
    """The sequential Model-API path on a fresh model: setRightHandSide / Equality.setRightHandSide / setCost."""
    from jslpsolver_b200.model import Equality
    m = _cpu_model(jm)
    m.tableau, m.tableauInitialized = _Recorder(), True
    for name, value in (spec.get("rhs") or {}).items():
        rows = [c for c in m.constraints if c.name == name]
        if isinstance(value, dict):
            for side, v in value.items():
                next(c for c in rows if c.isUpperBound == (side == "max")).setRightHandSide(v)
        elif len(rows) == 2:
            up, lo = sorted(rows, key=lambda c: not c.isUpperBound)
            Equality(up, lo).setRightHandSide(value)
        else:
            rows[0].setRightHandSide(value)
    for vid, value in (spec.get("cost") or {}).items():
        m.setCost(value, next(v for v in m.variables if v.id == vid))
    return m.tableau.calls


def _bits(edits):
    return [(k, i, np.float64(d).view(np.uint64)) for k, i, d in edits]


@pytest.mark.parametrize("op", ["max", "min"])
def test_edit_list_equals_the_model_api_path(op):
    from jslpsolver_b200.scenarios import edits_of
    jm = dict(EQ_MINMAX, opType=op)
    specs = [{}, {"rhs": {"mix": 12}}, {"rhs": {"mix": 10}}, {"rhs": {"band": {"max": 5, "min": 1}}},
             {"rhs": {"band": {"min": 2}}}, {"rhs": {"band": {"min": 5, "max": 5}}, "cost": {"w": 1, "x": 7}},
             {"cost": {"y": 2}}, {"cost": {"x": 3.5}, "rhs": {"cap": 29.75, "mix": 9.5}},
             {"rhs": {"cap": 30, "band": {"max": 8.0, "min": 2.5}}}]
    for spec in specs:
        m = _cpu_model(jm)
        before = ([c.rhs for c in m.constraints], [v.cost for v in m.variables])
        got = edits_of(m, spec)
        assert _bits(got) == _bits(_literal(jm, spec)), spec
        assert ([c.rhs for c in m.constraints], [v.cost for v in m.variables]) == before, "the model changed"
    # an unchanged right-hand side is skipped; an unchanged cost is not (setCost has no such test), and a max model
    # passes the negated difference, -0.0
    assert edits_of(_cpu_model(jm), {"rhs": {"mix": 10, "cap": 30}}) == []
    (k, i, d), = edits_of(_cpu_model(jm), {"cost": {"y": 2.0}})
    assert d == 0.0 and math.copysign(1.0, d) == (-1.0 if op == "max" else 1.0)
    # an equality moves its upper row, then its lower row; a min+max dict its rows in key order
    m = _cpu_model(jm)
    up = next(c for c in m.constraints if c.name == "mix" and c.isUpperBound)
    assert [e[1] for e in edits_of(m, {"rhs": {"mix": 3}})][0] == up.index
    band = {c.isUpperBound: c.index for c in m.constraints if c.name == "band"}
    assert [e[1] for e in edits_of(m, {"rhs": {"band": {"max": 7, "min": 1}}})] == [band[True], band[False]]
    assert [e[1] for e in edits_of(m, {"rhs": {"band": {"min": 1, "max": 7}}})] == [band[False], band[True]]


class _StubTableau:
    """Stands in for GpuTableau: runs the oracle definition of every scenario as the device batch would."""

    def __init__(self, model, sol):
        self.model, self.sol = model, sol
        self.handle = object()
        self._version = self._solved_version = 0
        self.precision = model.precision
        self.variablesPerIndex = model.variablesPerIndex
        self.evaluation = sol.state.evaluation if sol.state is not None else 0.0
        self.isIntegralFlag = None
        self.batches = 0

    def scenario_batch(self, edits, offsets):
        from oracle import scenarios as OS
        self.batches += 1
        out = {k: [] for k in ("status", "eval_raw", "p1", "p2", "rhs", "vrow")}
        for s in range(len(offsets) - 1):
            st, tab = OS.run(self.sol, edits[offsets[s]:offsets[s + 1]])
            M, (vrow, _) = tab.matrix(), tab.maps()
            out["status"].append(3 if st.cyclePhase else 1 if not st.feasible else 2 if not st.bounded else 0)
            out["eval_raw"].append(M[0, 0])
            out["p1"].append(st.lastP1)
            out["p2"].append(st.lastP2)
            out["rhs"].append(M[:, 0].copy())
            out["vrow"].append(vrow)
        return out


def _solution(jm, feasible=None, bounded=None):
    from jslpsolver_b200.tableau import Solution
    from oracle import ref_model
    sol = ref_model.solve_full(jm, fast_cycles=True)
    m = _cpu_model(jm)
    t = _StubTableau(m, sol)
    return Solution(t, sol.evaluation, sol.feasible if feasible is None else feasible,
                    sol.bounded if bounded is None else bounded)


def test_berlin_airlift_known_answers():
    """README's parametric() answers as scenarios: person 352 -> 880 000; person 0 -> 0; brit's cost 40 000 ->
    1 760 000 with brit = 44; no edit -> the solved result."""
    sol = _solution(BERLIN)
    out = sol.scenarios([{"rhs": {"person": 352}}, {"rhs": {"person": 0}}, {"cost": {"brit": 40000}}, {}])
    assert out[0]["result"] == 880000.0 and out[0]["feasible"] and out[0]["bounded"]
    assert out[1]["result"] == 0 and out[1]["feasible"]
    assert out[2]["result"] == 1760000.0 and out[2]["brit"] == 44.0 and "yank" not in out[2]
    from oracle import ref_model
    assert out[3] == ref_model.Solve(BERLIN)
    assert sol.scenarios([]) == [] and sol._tableau.batches == 1


@pytest.mark.parametrize("fx", [f for f in CONTINUOUS if f["file"] != "Monster Problem.json"], ids=lambda f: f["file"])
def test_host_results_equal_the_oracle_definition(fx):
    """Solution.scenarios() over the oracle definition equals oracle/scenarios.result key for key and bit for bit
    (presolve as Solve() runs it)."""
    from jslpsolver_b200.scenarios import edits_of
    from oracle import ref_model
    from oracle import scenarios as OS
    jm = strip_timeouts(fx["model"])
    osol = ref_model.solve_full(jm, fast_cycles=True)
    if osol.tableau is None or not (osol.feasible and osol.bounded):
        pytest.skip("no optimum")
    sol = _solution(jm)
    m = sol._tableau.model
    fixed = m.presolveResult.fixedVariables
    specs = [dict(s, cost={k: v for k, v in s["cost"].items() if next(x for x in m.variables if x.id == k) not in fixed})
             for s in _perturbations(jm, m, osol, 6, seed=3)]
    got = sol.scenarios(specs)
    for spec, g in zip(specs, got):
        want = OS.result(osol, edits_of(m, spec))
        assert list(g) == list(want) and all(np.float64(g[k]).tobytes() == np.float64(want[k]).tobytes()
                                             for k in g if not isinstance(g[k], bool)), (spec, g, want)


def test_value_errors():
    from jslpsolver_b200.tableau import Solution
    jm = dict(BERLIN, constraints=dict(BERLIN["constraints"], labor={"min": 1, "max": 50}),
              variables={k: dict(v, labor=1) for k, v in BERLIN["variables"].items()})
    sol = _solution(jm)
    for cases, match in (([{"rhs": {"nope": 1}}], "no constraint named"), ([{"cost": {"nope": 1}}], "no variable named"),
                         ([{"rhs": {"labor": 3}}], "min and a max bound"), ([{"rhs": {"person": {"min": 3}}}], "only a 'max'"),
                         ([{"rhs": {"labor": {"lo": 3}}}], "side must be"), ([{"rhs": {"labor": {}}}], "needs a 'min'"),
                         ([{"rhs": {"person": math.nan}}], "finite number"), ([{"rhs": {"person": math.inf}}], "finite"),
                         ([{"cost": {"brit": -math.inf}}], "finite"), ([{"rhs": {"person": True}}], "finite"),
                         ([{"rhs": {"person": "3"}}], "finite"), ([{"rhs": {"labor": {"max": math.nan}}}], "finite"),
                         ([{"rhs": {"person": 1}, "coefficients": {}}], "unknown scenario key"), ([3], "a scenario is a dict"),
                         ([{"rhs": [("person", 1)]}], "must be a dict"), ({"rhs": {}}, "takes a list"),
                         ([{}, {"rhs": {"nope": 1}}], "no constraint named")):
        with pytest.raises(ValueError, match=match):
            sol.scenarios(cases)
    assert sol._tableau.batches == 0, "a refused call ran scenarios"
    # the cases sensitivity() refuses, with scenarios() named in the message
    lp0 = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Berlin Air Lift Problem.json"][0]["model"])
    mip = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Integer Berlin Air Lift Problem.json"][0]["model"])
    soft = dict(lp0, constraints=dict(lp0["constraints"], plane={"max": 44, "weight": 10}))
    for model, feasible, bounded, match in ((mip, True, True, "integer or binary"), (soft, True, True, "soft constraints"),
                                            (lp0, False, True, "infeasible"), (lp0, True, False, "unbounded")):
        with pytest.raises(ValueError, match=r"scenarios\(\).*" + match):
            _solution(model, feasible, bounded).scenarios([{}])
    s = _solution(lp0)
    s._tableau._version += 1
    with pytest.raises(ValueError, match="edited or solved again"):
        s.scenarios([{}])
    s._tableau.handle = None
    with pytest.raises(ValueError, match="has not been solved"):
        Solution(s._tableau, 0.0, True, True).scenarios([{}])
    # -x <= -2 and x <= 2: presolve fixes x = 2
    fixed = {"optimize": "z", "opType": "max", "constraints": {"lo": {"max": -2}, "hi": {"max": 2}, "cap": {"max": 7}},
             "variables": {"x": {"z": 1, "lo": -1, "hi": 1, "cap": 1}, "y": {"z": 2, "cap": 1}}}
    sf = _solution(fixed)
    assert sf._tableau.model.presolveResult.fixedVariables, "presolve fixes x"
    with pytest.raises(ValueError, match=r"scenarios\(\): presolve fixed 'x' and zeroed its cost"):
        sf.scenarios([{"cost": {"x": 3}}])
    assert sf.scenarios([{"cost": {"y": 3}}])[0]["result"] == 15.0


def test_ctypes_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    st = re.search(r"typedef struct \{([^}]*)\}\s*jslp_scenario_edit\s*;", header)
    assert st, "jslp_scenario_edit is not declared"
    fields = [tuple(f.split()) for f in st.group(1).replace("\n", " ").split(";") if f.strip()]
    assert fields == [("int32_t", "kind"), ("int32_t", "index"), ("double", "difference")], fields
    C = _lib.C
    assert [(n, t) for n, t in _lib.ScenarioEdit._fields_] == [("kind", C.c_int32), ("index", C.c_int32),
                                                               ("difference", C.c_double)]
    assert C.sizeof(_lib.ScenarioEdit) == 16
    proto = re.search(r"\bint\s+jslp_scenario_batch\s*\(([^)]*)\)\s*;", header)
    assert proto, "jslp_scenario_batch is not declared"
    params = [re.sub(r"\s+", " ", p.strip()) for p in proto.group(1).split(",")]
    types = [re.sub(r"\s*\b\w+$", "", p).replace(" *", "*") for p in params]
    want = ["jslp_tab*", "const jslp_scenario_edit*", "const int32_t*", "int", "int", "int32_t*", "double*", "int32_t*",
            "int32_t*", "double*", "int32_t*"]
    assert types == want, types
    (name, res, args), = [s for s in _lib.SYMBOLS if s[0] == "jslp_scenario_batch"]
    assert res is C.c_int and len(args) == len(want)
    for a, w in zip(args, want):
        assert (a is C.c_void_p) if w.endswith("*") else (a is C.c_int), (w, a)

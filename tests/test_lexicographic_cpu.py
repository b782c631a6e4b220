"""CPU checks of lexicographic objectives (DESIGN.md section 2j) over the restatement in lexicographic_oracle.py: at
every level the optimum equals SciPy HiGHS's optimum of that objective over the model's rows plus `objective_j >= z_j
- t_j` (max) / `<= z_j + t_j` (min) for every earlier level j, and the final plan is feasible and within every t_j of
z_j -- on the continuous fixtures with seeded extra objectives, seeded alternative_optima_multi_model chains of 2, 3 and
5 levels, dense_packing_multi_model, mixed_lp_model with extra objectives, a presolve-fixed variable, an unbounded
second level, an infeasible model and a single-point face.  Also: level 1 is Solve(full=True) of the first objective,
the zero-allowance chain of two objectives ends at the last frontier vertex, a huge allowance makes level 2 the second
objective alone, later optima are monotone in the gap, no level after the first makes a phase-1 pivot, the host driver
over a stand-in tableau equals the restatement, every refusal, the gap validation and the C prototype."""
import math
import os
import re
import types

import numpy as np
import pytest

import lexicographic_oracle as LO
import near_optimal_oracle as NO
import test_variability_cpu as TV
from conftest import ROOT, load_bundle
from helpers import strip_timeouts

BUNDLE = load_bundle()
P = 1e-8
BERLIN = {"optimize": {"capacity": "max", "cost": "min"},
          "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
          "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                        "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}
FIXTURES = [f for f in TV.CONTINUOUS]


def _with_extra(jm, senses, seed, lo=0, hi=20):
    """jm with seeded extra objectives extra1.. of the given senses after its own objective."""
    rng = np.random.default_rng(seed)
    jm = strip_timeouts(jm)
    names = [f"extra{k + 1}" for k in range(len(senses))]
    for v in jm["variables"].values():
        for n in names:
            v[n] = float(rng.integers(lo, hi + 1))
    return dict(jm, optimize={jm["optimize"]: "max" if jm.get("opType") == "max" else "min",
                              **dict(zip(names, senses))})


class _Highs:
    """The JSON model as A x <= b, x >= 0 with one objective vector per `optimize` key."""

    def __init__(self, jm):
        from scipy.optimize import linprog
        self.linprog = linprog
        self.names = list(jm["variables"])
        rows = TV._rows(jm, self.names)
        self.A = np.array([a if kind == "max" else -a for _, kind, a, _ in rows])
        self.b = np.array([b if kind == "max" else -b for _, kind, _, b in rows])
        self.keys = list(jm["optimize"])
        self.sense = {k: jm["optimize"][k] for k in self.keys}
        self.c = {k: np.array([float(jm["variables"][v].get(k) or 0.0) for v in self.names]) for k in self.keys}

    def _bounds(self, upto, opt, allow):
        A, b = [self.A], list(self.b)
        for j in range(upto):
            key = self.keys[j]
            if self.sense[key] == "max":  # c.x >= z - t
                A.append(-self.c[key][None, :]); b.append(-(opt[j] - allow[j]))
            else:
                A.append(self.c[key][None, :]); b.append(opt[j] + allow[j])
        return np.vstack(A), np.array(b)

    def level(self, k, opt, allow):
        """HiGHS's optimum of objective k over the rows and the bounds of levels 0..k-1; +-inf when unbounded."""
        A, b = self._bounds(k, opt, allow)
        key = self.keys[k]
        s = 1.0 if self.sense[key] == "max" else -1.0
        res = self.linprog(-s * self.c[key], A_ub=A, b_ub=b, bounds=(0, None), method="highs")
        if res.status == 3:
            return s * math.inf
        assert res.status == 0, res.message
        return -s * res.fun

    def check_plan(self, x, opt, allow, tol=1e-7):
        x = np.array([x[v] for v in self.names])
        scale = max(1.0, float(np.abs(x).max(initial=0.0)))
        assert (x >= -tol * scale).all()
        assert (self.A @ x <= self.b + tol * np.maximum(1.0, np.abs(self.b)) * scale).all()
        for j in range(len(opt)):
            key = self.keys[j]
            loss = (opt[j] - self.c[key] @ x) if self.sense[key] == "max" else (self.c[key] @ x - opt[j])
            assert loss <= allow[j] + tol * max(1.0, abs(opt[j])) * scale, (key, loss, allow[j])


def _const(jm, key, fixed):
    """What the variables presolve fixed add to objective `key` (the tableau's objectives leave them out)."""
    return sum(float(jm["variables"][vid].get(key) or 0.0) * x for vid, x in fixed.items())


def check_chain(jm, gap=0.0, absolute_gap=0.0):
    """The restatement of jm against HiGHS level by level; returns (result, details)."""
    jm = strip_timeouts(jm)
    res, det = LO.chain(jm, gap, absolute_gap)
    if not res["feasible"]:
        return res, det
    h = _Highs(jm)
    fixed = det[0]["fixed"]
    for d in det[1:]:
        assert d["p1"] == 0, "a level after the first made a phase-1 pivot"
    opt, allow = [], []
    for k, lv in enumerate(res["levels"]):
        if lv["optimum"] is None:
            assert res["stop"] in ("unbounded", "cycled") and k == len(res["levels"]) - 1
            if res["stop"] == "unbounded":
                assert math.isinf(h.level(k, opt, allow)), (k, "HiGHS finds a bounded level")
            break
        z = lv["optimum"] + _const(jm, lv["objective"], fixed)
        want = h.level(k, opt, allow)
        assert TV._close(z, want), (k, lv["objective"], z, want)
        opt.append(z)
        allow.append(lv["allowance"] if lv["allowance"] is not None else 0.0)
    if res["values"] is not None:
        h.check_plan(res["values"], opt[:-1] if res["stop"] == "reached" else opt, allow)
    return res, det


# ---------------------------------------------------------------- against HiGHS
@pytest.mark.parametrize("fx", FIXTURES, ids=lambda f: f["file"])
def test_fixture_chains_match_highs(fx):
    """Every continuous fixture without unrestricted variables with two seeded extra objectives of mixed senses; the
    600-row fixture at one setting only."""
    pytest.importorskip("scipy")
    big = len(fx["model"]["constraints"]) > 100
    for gap in ((0.01,) if big else (0.0, 0.01)):
        res, _ = check_chain(_with_extra(fx["model"], ["min", "max"], seed=3), gap=gap)
        if not res["feasible"]:
            pytest.skip("infeasible")


@pytest.mark.parametrize("levels", [2, 3, 5])
@pytest.mark.parametrize("seed", range(3))
def test_alternative_optima_chains_match_highs(levels, seed):
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    jm = problems.alternative_optima_multi_model(18 + seed, 9 + seed, levels, seed=30 + seed)
    kinds = set()
    for gap, absolute_gap in ((0.0, 0.0), (0.01, 0.0), (0.0, 2.0), ({"objective": 0.02}, {"obj1": 1.0})):
        res, _ = check_chain(jm, gap, absolute_gap)
        assert res["stop"] == "reached" and len(res["levels"]) == levels
        kinds |= {lv["kind"] for lv in res["levels"][1:]}
    assert {"face", "bound"} <= kinds, kinds


def test_dense_packing_and_mixed_chains_match_highs():
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    for seed in range(2):
        for gap in (0.0, 0.005):
            check_chain(problems.dense_packing_multi_model(14 + seed, 10 + seed, 3, seed=50 + seed), gap=gap)
    checked = 0
    for k in range(30):
        jm = _with_extra(problems.mixed_lp_model(10, 8, seed=700 + k), ["max", "min", "max"], seed=k)
        res, _ = check_chain(jm, gap=0.01)
        checked += res["feasible"] and res["stop"] == "reached"
        if checked >= 3:
            return
    pytest.fail(f"only {checked} seeded mixed LPs reached the last level")


def test_presolve_fixed_unbounded_infeasible_and_single_point():
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    fixed = {"optimize": {"z": "max", "w2": "min"},
             "constraints": {"lo": {"max": -2}, "hi": {"max": 2}, "cap": {"max": 7}},
             "variables": {"x": {"z": 1, "w2": 5, "lo": -1, "hi": 1, "cap": 1}, "y": {"z": 2, "w2": 1, "cap": 1},
                           "w": {"z": 2, "w2": 3, "cap": 1}}}
    for absolute_gap in (0.0, 3.0):
        res, det = check_chain(fixed, absolute_gap=absolute_gap)
        assert det[0]["fixed"] == {"x": 2} and res["values"]["x"] == 2 and res["stop"] == "reached"
    # max x s.t. x <= 5, then max y with x - y <= 2 only: the second level runs off
    ray = {"optimize": {"a": "max", "b": "max"}, "constraints": {"gap": {"max": 2}, "cap": {"max": 5}},
           "variables": {"x": {"a": 1, "gap": 1, "cap": 1}, "y": {"b": 1, "gap": -1}}}
    res, det = check_chain(ray)
    assert res["stop"] == "unbounded" and not res["bounded"] and res["levels"][1]["optimum"] is None
    assert res["values"]["x"] == 5.0 and res["levels"][0]["optimum"] == 5.0
    first = dict(ray, optimize={"b": "max", "a": "max"})
    res, _ = check_chain(first)
    assert res["stop"] == "unbounded" and res["values"] is None and res["objectives"] is None
    assert len(res["levels"]) == 1
    res, _ = check_chain(dict(problems.planted_infeasible_model(8, 6, 2, seed=4), optimize={"objective": "max", "b": "max"}))
    assert not res["feasible"] and len(res["levels"]) == 1 and res["values"] is None
    # Berlin Airlift: no reduced cost is 0 at the capacity optimum, so its face is the optimum alone
    res, det = check_chain(dict(BERLIN, optimize={"capacity": "max", "cost": "min", "plane": "max"}))
    assert [lv["kind"] for lv in res["levels"]] == ["solve", None, None] and len(det) == 1
    assert res["levels"][1]["optimum"] == res["objectives"]["cost"] and res["stop"] == "reached"


# ---------------------------------------------------------------- properties
def test_level_one_is_solve_of_the_first_objective():
    from jslpsolver_b200 import problems
    from oracle import ref_model
    for jm in (BERLIN, problems.alternative_optima_multi_model(20, 10, 3, seed=1)):
        res, det = LO.chain(jm, 0.01)
        keys = list(jm["optimize"])
        sol = ref_model.solve_full(dict(jm, optimize=keys[0], opType=jm["optimize"][keys[0]]))
        M = sol.tableau.matrix()
        assert np.array_equal(det[0]["M"].view(np.uint64), M.view(np.uint64))
        assert (det[0]["p1"], det[0]["p2"]) == (sol.state.lastP1, sol.state.lastP2)
        sigma = 1.0 if jm["optimize"][keys[0]] == "max" else -1.0
        assert res["levels"][0]["optimum"] == -sigma * M[0, 0] + 0.0
        assert abs(res["levels"][0]["optimum"] - sol.evaluation) <= 1e-8 * max(1.0, abs(sol.evaluation))  # Solve rounds


def test_zero_allowance_ends_at_the_last_frontier_vertex():
    """By section 2g the last vertex of Frontier({a, b}) is the lexicographic optimum, b first and then a."""
    from jslpsolver_b200 import problems
    from oracle import frontier as OF
    cases = [BERLIN, problems.dense_packing_multi_model(12, 9, 2, seed=3),
             problems.alternative_optima_multi_model(16, 8, 2, seed=5)]
    for jm in cases:
        a, b = list(jm["optimize"])
        fr, _ = OF.Frontier(jm)
        lex, _ = LO.chain(dict(jm, optimize={b: jm["optimize"][b], a: jm["optimize"][a]}))
        want = fr["vertices"][-1]["objectives"]
        for key in (a, b):
            assert abs(lex["objectives"][key] - want[key]) <= 1e-9 * max(1.0, abs(want[key])), (key, lex, want)


def test_huge_allowance_is_the_second_objective_alone():
    from jslpsolver_b200 import problems
    from oracle import ref_model
    jm = problems.alternative_optima_multi_model(20, 10, 2, seed=2)
    res, _ = LO.chain(jm, absolute_gap=1e9)
    alone = ref_model.solve_full(dict(jm, optimize="obj1", opType="min"))
    assert TV._close(res["levels"][1]["optimum"], alone.evaluation, 1e-9)


def test_later_optima_are_monotone_in_the_gap():
    from jslpsolver_b200 import problems
    jm = problems.alternative_optima_multi_model(24, 12, 3, seed=8)
    prev = None
    for gap in (0.0, 1e-4, 1e-3, 1e-2, 0.05, 0.2):
        res, det = LO.chain(jm, gap)
        assert all(d["p1"] == 0 for d in det[1:])
        z2 = res["levels"][1]["optimum"]  # obj1 is a min: it can only fall as level 1 gives up more
        if prev is not None:
            assert z2 <= prev + 1e-9 * max(1.0, abs(prev)), (gap, z2, prev)
        prev = z2


def test_child_row_zero_is_the_frontier_pricing():
    """Rule 2 on a solved seeded optimum: row 0 of the child is oracle.frontier.price at the kept columns, every other
    element is the face's or the bound tableau's."""
    from jslpsolver_b200 import problems
    from oracle import frontier as OF
    from oracle import variability as OV
    jm = problems.alternative_optima_multi_model(20, 10, 2, seed=4)
    res, det = LO.chain(jm, 0.0)
    M, vrow, vcol = det[0]["M"], det[0]["vrow_f"], det[0]["vcol_f"]
    c = det[1]["cost"]
    R = OF.price(M, vrow, vcol, c)[0]
    bits = lambda a: np.ascontiguousarray(a).view(np.uint64)  # noqa: E731
    kept, F, vcol_f = OV.face(M, vcol, P)
    T, vr, vc, k2 = LO.child(M, vrow, vcol, P, c, 0.0, 99)
    assert np.array_equal(k2, kept) and np.array_equal(bits(T[1:]), bits(F[1:])) and np.array_equal(vc, vcol_f)
    assert np.array_equal(bits(T[0]), bits(R[kept]))
    n = M.shape[0] + M.shape[1] - 2
    T, vr, vc, k2 = LO.child(M, vrow, vcol, P, c, 2.5, n)
    B, vrow_b, _ = NO.bound(M, vrow, vcol, 2.5, n)
    assert np.array_equal(bits(T[1:]), bits(B[1:])) and np.array_equal(bits(T[0]), bits(R))
    assert list(vr) == list(vrow_b) and list(k2) == list(range(M.shape[1]))


# ---------------------------------------------------------------- the host driver over a stand-in tableau
class _StubTab:
    """Stands in for GpuTableau over the restatement: lex_next builds rule 2's tableau, simplex runs rule 3."""

    def __init__(self, log, M, vrow, vcol, n, status=None):
        self.log, self.M, self.vrow, self.vcol, self.nVars = log, M, vrow, vcol, n
        self.height, self.width = M.shape
        self.lastStatus = status
        self.feasible = self.bounded = True
        self.closed = False

    def lex_next(self, cost, t):
        assert not self.closed and len(cost) == self.nVars
        self.log.append(("lex_next", t))
        T, vr, vc, kept = LO.child(self.M, self.vrow, self.vcol, P, np.asarray(cost, dtype=np.float64), t,
                                   NO.fresh_label(self.nVars, self.nVars))
        if T is None:
            return None, kept
        return _StubTab(self.log, T, vr, vc, self.nVars + (t > 0.0)), kept

    def simplex(self, check_cycles=None):
        assert check_cycles is True
        status, p1, p2, self.M, self.vrow, self.vcol = LO.solve(self.M, self.vrow, self.vcol, P)
        self.lastStatus = types.SimpleNamespace(phase1_pivots=p1, phase2_pivots=p2, cycled=int(status == LO.CYCLED))
        self.feasible, self.bounded = status != LO.INFEASIBLE, status != LO.UNBOUNDED
        return self

    def final_state(self):
        return self.M[:, 0].copy(), self.M[0].copy(), self.vrow, self.vcol

    def close(self):
        self.closed = True
        self.log.append(("close",))


class _StubSolver:
    def __init__(self):
        self.log, self.tabs = [], []

    def _instance(self, working, precision):
        from oracle import ref_model
        sol = ref_model.solve_full(working, precision)
        m = TV._cpu_model(working)
        if sol.tableau is None:
            tab = types.SimpleNamespace(lastStatus=None, width=0, height=0)
        else:
            M = sol.tableau.matrix()
            vrow, vcol = sol.tableau.maps()
            st = types.SimpleNamespace(phase1_pivots=sol.state.lastP1, phase2_pivots=sol.state.lastP2,
                                       cycled=int(bool(sol.state.cyclePhase)))
            tab = _StubTab(self.log, M, vrow, vcol, M.shape[0] + M.shape[1] - 2, st)
            tab.feasible, tab.bounded = sol.feasible, sol.bounded
        m.tableau = tab
        m.solve = lambda: types.SimpleNamespace(feasible=sol.feasible, bounded=sol.bounded)
        return m


def _host(jm, gap=0.0, absolute_gap=0.0):
    from jslpsolver_b200.lexicographic import Lexicographic
    s = _StubSolver()
    return Lexicographic(s, jm, gap, absolute_gap), s.log


def test_host_driver_equals_the_restatement():
    from jslpsolver_b200 import problems
    cases = [(problems.alternative_optima_multi_model(18, 9, 3, seed=1), 0.0, 0.0),
             (problems.alternative_optima_multi_model(18, 9, 5, seed=2), 0.01, 0.0),
             (problems.alternative_optima_multi_model(18, 9, 4, seed=3), {"objective": 0.01}, {"obj2": 3.0}),
             (problems.dense_packing_multi_model(12, 9, 3, seed=3), 0.002, 0.0),
             (dict(BERLIN, optimize={"capacity": "max", "cost": "min", "plane": "max"}), 0.0, 0.0),
             ({"optimize": {"a": "max", "b": "max"}, "constraints": {"gap": {"max": 2}, "cap": {"max": 5}},
               "variables": {"x": {"a": 1, "gap": 1, "cap": 1}, "y": {"b": 1, "gap": -1}}}, 0.0, 1.0),
             (dict(problems.planted_infeasible_model(8, 6, 2, seed=4), optimize={"objective": "max", "b": "max"}), 0.0, 0.0)]
    for jm, gap, absolute_gap in cases:
        want, _ = LO.chain(jm, gap, absolute_gap)
        got, log = _host(jm, gap, absolute_gap)
        assert got == want, (jm.get("name"), got, want)
        # only the current child stays alive: each is closed once the next exists, the last one at the end
        made = sum(1 for e in log if e[0] == "lex_next")
        ran = sum(1 for lv in got["levels"][1:] if lv["kind"] is not None)
        assert sum(1 for e in log if e[0] == "close") == ran, log
        assert made >= ran


def test_refusals_and_gap_validation():
    from jslpsolver_b200.lexicographic import Lexicographic
    s = _StubSolver()
    one = dict(BERLIN, optimize={"capacity": "max"})
    for model, match in ((one, "at least two"), (dict(BERLIN, optimize="capacity"), "at least two"),
                         (dict(BERLIN, ints={"brit": 1}), "integer or binary"),
                         (dict(BERLIN, binaries={"yank": 1}), "integer or binary"),
                         (dict(BERLIN, constraints=dict(BERLIN["constraints"], plane={"max": 44, "weight": 3})), "soft"),
                         (dict(BERLIN, constraints=dict(BERLIN["constraints"], plane={"max": 44, "priority": "strong"})),
                          "soft"),
                         (dict(BERLIN, unrestricted={"brit": 1}), "unrestricted variables: re-solving from an optimum")):
        with pytest.raises(ValueError, match=r"Lexicographic\(\).*" + re.escape(match)):
            Lexicographic(s, model)
    with pytest.raises(NotImplementedError):
        Lexicographic(s, dict(BERLIN, external={"solver": "x"}))
    for kw, match in (({"gap": -0.01}, "gap= must be finite and >= 0"), ({"gap": math.nan}, "gap= must be finite"),
                      ({"gap": math.inf}, "gap= must be finite"), ({"absolute_gap": -1}, "absolute_gap= must be"),
                      ({"absolute_gap": -math.inf}, "absolute_gap="), ({"gap": "1%"}, "gap= takes a number"),
                      ({"gap": None}, "gap= takes a number"), ({"absolute_gap": True}, "absolute_gap= takes a number"),
                      ({"gap": [0.1]}, "gap= takes a number"), ({"gap": {"capacity": False}}, "gap= takes a number"),
                      ({"gap": {"capacity": -1.0}}, "gap= must be"), ({"gap": {"nope": 0.1}}, "names 'nope'"),
                      ({"absolute_gap": {"plane": 1.0}}, "names 'plane'"), ({"gap": 1e308}, "overflows")):
        with pytest.raises(ValueError, match=r"Lexicographic\(\).*" + re.escape(match)):
            Lexicographic(s, BERLIN, **kw)
    assert not any(e[0] == "lex_next" for e in s.log), "a refused call built a level"
    res = Lexicographic(s, BERLIN, gap=np.float64(0.01))
    assert res["levels"][0]["allowance"] == 0.01 * 1080000.0


def test_ctypes_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    import jslpsolver_b200 as J
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+jslp_lex_next\s*\(([^)]*)\)\s*;", header)
    assert proto, "jslp_lex_next is not declared"
    params = [re.sub(r"\s+", " ", p.strip()) for p in proto.group(1).split(",")]
    types_ = [re.sub(r"\s*\b\w+$", "", p).replace(" *", "*") for p in params]
    assert types_ == ["jslp_tab*", "const double*", "double", "jslp_tab**", "int32_t*", "int32_t*"], types_
    assert "section 2j" in header[:proto.start()][-1500:]
    (name, res, args), = [s for s in _lib.SYMBOLS if s[0] == "jslp_lex_next"]
    C = _lib.C
    assert res is C.c_int and len(args) == 6 and args[0] is C.c_void_p and args[1] is C.c_void_p
    assert args[2] is C.c_double and args[3]._type_ is C.c_void_p and args[4]._type_ is C.c_int32
    assert args[5] is C.c_void_p
    src = open(os.path.join(ROOT, "jslpsolver_b200", "csrc", "jslp_api.cu")).read()
    assert '#include "jslp_lex.cuh"' in src.split('#include "jslp_bound.cuh"')[1]
    assert J.Lexicographic is not None and J.Solver.Lexicographic is not None and "Lexicographic" in J.__all__

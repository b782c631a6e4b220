"""CPU checks of the sensitivity report (DESIGN.md section 2b) on final tableaux from the oracle: duals and reduced
costs against SciPy's HiGHS, ranges by re-solving perturbed LPs, hand-derived answers for the Berlin Airlift, the host
mirror's assembly against the oracle's restatement, its ValueError cases, and the C prototype against ctypes."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_bundle
from helpers import strip_timeouts

BUNDLE = load_bundle()


def _fixture(name):
    return strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == name][0]["model"])


def _rel(a, b, tol=1e-9):
    return abs(a - b) <= tol * max(1.0, abs(b))


def _random_lp(rng, with_equal):
    """A feasible, bounded LP around an interior point x0: random dense rows of every kind the caller allows, costs of
    either sign, either sense, and a `cap` row (sum x <= ...) that bounds every variable."""
    n, m = int(rng.integers(2, 7)), int(rng.integers(2, 7))
    x0 = rng.uniform(1.0, 5.0, n)
    kinds = ["max", "min", "equal"] if with_equal else ["max", "min"]
    constraints, rows = {}, {}
    for i in range(m):
        a = np.round(rng.uniform(-2.0, 5.0, n), 3)
        kind = kinds[int(rng.integers(0, len(kinds)))]
        b = float(a @ x0)
        b = round(b + rng.uniform(0.5, 4.0), 3) if kind == "max" else round(b - rng.uniform(0.5, 4.0), 3) if kind == "min" else b
        constraints[f"c{i}"] = {kind: b}
        rows[f"c{i}"] = a
    constraints["cap"] = {"max": round(float(x0.sum()) + rng.uniform(1.0, 10.0), 3)}
    rows["cap"] = np.ones(n)
    cost = np.round(rng.uniform(-10.0, 10.0, n), 3)
    variables = {f"x{j}": {"obj": float(cost[j]), **{r: float(a[j]) for r, a in rows.items()}} for j in range(n)}
    return {"optimize": "obj", "opType": "max" if rng.random() < 0.5 else "min", "constraints": constraints,
            "variables": variables}


def _degenerate(sol, jm, tol=1e-7):
    """A basic variable at zero or a non-basic column with a zero reduced cost: the duals or the optimal basis are not
    unique.  An equality's two rows leave at least one of their slacks basic at zero; one such slack per equality is
    not counted (both basic would leave the equality's dual undetermined)."""
    from oracle import sensitivity as S
    M = sol.tableau.matrix()
    vrow, _ = sol.tableau.maps()
    names = S.json_row_names(jm)
    equality = {con.index: names[k] for k, con in enumerate(sol.model.constraints)
                if k < len(names) and jm["constraints"][names[k]].get("equal") is not None}
    zeros = [int(vrow[r]) for r in range(1, M.shape[0]) if abs(M[r, 0]) <= tol]
    pairs = [equality[v] for v in zeros if v in equality]
    primal = len(zeros) > len(pairs) or len(pairs) != len(set(pairs))
    dual = bool(np.any(np.abs(M[0, 1:]) <= tol))
    return primal or dual


def _highs(jm):
    """linprog(HiGHS) of jm: (result, {row name: d result / d rhs}, {var: d result / d x_j at its bound 0})."""
    from scipy.optimize import linprog
    names = list(jm["variables"])
    kappa = -1.0 if jm["opType"] == "max" else 1.0   # result = kappa * fun
    c = kappa * np.array([jm["variables"][v].get(jm["optimize"], 0.0) for v in names])
    A_ub, b_ub, ub_rows, A_eq, b_eq, eq_rows = [], [], [], [], [], []
    for cname, spec in jm["constraints"].items():
        a = np.array([jm["variables"][v].get(cname, 0.0) for v in names])
        if "equal" in spec:
            A_eq.append(a); b_eq.append(spec["equal"]); eq_rows.append(cname)
        elif "max" in spec:
            A_ub.append(a); b_ub.append(spec["max"]); ub_rows.append((cname, 1.0))
        else:
            A_ub.append(-a); b_ub.append(-spec["min"]); ub_rows.append((cname, -1.0))
    res = linprog(c, A_ub=np.array(A_ub) if A_ub else None, b_ub=b_ub or None, A_eq=np.array(A_eq) if A_eq else None,
                  b_eq=b_eq or None, bounds=(0, None), method="highs")
    assert res.status == 0, res.message
    duals = {}
    for (cname, s), mg in zip(ub_rows, res.ineqlin.marginals):
        duals[cname] = duals.get(cname, 0.0) + kappa * s * mg
    for cname, mg in zip(eq_rows, res.eqlin.marginals):
        duals[cname] = duals.get(cname, 0.0) + kappa * mg
    return kappa * res.fun, duals, {v: kappa * mg for v, mg in zip(names, res.lower.marginals)}


def test_duals_and_reduced_costs_match_highs():
    """>= 100 random nondegenerate LPs (max / min / equal rows, both senses, costs of either sign): every dual and
    reduced cost equals the marginal HiGHS reports, converted to d result / d rhs and d result / d x_j."""
    pytest.importorskip("scipy")
    from oracle import ref_model
    from oracle import sensitivity as S
    rng = np.random.default_rng(2026)
    checked = skipped = 0
    seen = {"max": 0, "min": 0, "equal": 0, "sense max": 0, "sense min": 0}
    while checked < 100:
        jm = _random_lp(rng, with_equal=True)
        sol = ref_model.solve_full(jm)
        assert sol.feasible and sol.bounded
        if _degenerate(sol, jm):
            skipped += 1
            continue
        rep = S.report(jm, sol)
        result, duals, reduced = _highs(jm)
        raw = (1.0 if sol.model.isMinimization else -1.0) * sol.tableau.matrix()[0, 0]  # unrounded result
        assert _rel(raw, result), (raw, result)
        for name, d in rep["duals"].items():
            assert _rel(d, duals[name]), (jm, name, d, duals[name])
        for vid, v in rep["variables"].items():
            assert _rel(v["reducedCost"], reduced[vid]), (jm, vid, v["reducedCost"], reduced[vid])
        for spec in jm["constraints"].values():
            seen.update({k: seen[k] + 1 for k in spec})
        seen["sense " + jm["opType"]] += 1
        checked += 1
    assert skipped < checked and min(seen.values()) >= 10, (skipped, seen)


def _initial(jm):
    from oracle import ref_model
    model = ref_model.RefModel().loadJson(jm)
    M, vrow, vcol, _, _ = model.build_tableau()
    return model, M, vrow, vcol


def _solve_tableau(M, vrow, vcol):
    """(optimal?, basis as a set of variable indices, result) of the LP whose initial tableau is M (maximisation
    sense is read from the caller's sigma when the result is formed)."""
    from oracle import ref_model
    t = ref_model.OracleTableau(M, vrow, vcol)
    st = t.simplex()
    return bool(st.feasible and st.bounded), set(int(v) for v in t.maps()[0][1:]), t.matrix()[0, 0]


def test_ranges_by_perturbation():
    """Every finite range end of every row and variable, on nondegenerate LPs: half-way to the end the re-solved LP keeps
    the basis and `result` moves by dual * delta (value * delta for a cost); just beyond the end (1e-3 of the range
    width) the basis changes or the LP stops having an optimum."""
    from oracle import ref_model
    from oracle import sensitivity as S
    rng = np.random.default_rng(99)
    lps = ends = 0
    while lps < 30:
        jm = _random_lp(rng, with_equal=False)
        sol = ref_model.solve_full(jm)
        if _degenerate(sol, jm):
            continue
        rep = S.report(jm, sol)
        model, M0, vrow0, vcol0 = _initial(jm)
        sigma = -1.0 if model.isMinimization else 1.0
        ok, basis, raw = _solve_tableau(M0, vrow0, vcol0)
        assert ok
        result = -sigma * raw
        cases = []  # (current, range, slope, apply(M, new value))
        for i, (con, row) in enumerate(zip(model.constraints, rep["constraints"]), start=1):
            s = 1.0 if con.isUpperBound else -1.0
            cases.append((con.rhs, row["range"], row["dual"], lambda M, x, i=i, s=s: M.__setitem__((i, 0), s * x)))
        for j, var in enumerate(model.variables, start=1):
            v = rep["variables"][var.id]
            cases.append((var.cost, v["range"], v["value"], lambda M, x, j=j: M.__setitem__((0, j), sigma * x)))
        for cur, rng_, slope, apply in cases:
            lo, hi = rng_["min"], rng_["max"]
            assert lo <= cur <= hi or _rel(lo, cur) or _rel(hi, cur), (cur, rng_)
            width = hi - lo if np.isfinite(hi - lo) and hi > lo else None
            for end, out in ((lo, -1.0), (hi, 1.0)):
                if not np.isfinite(end):
                    continue
                ends += 1
                if end != cur:
                    M = M0.copy()
                    mid = cur + (end - cur) / 2
                    apply(M, mid)
                    ok2, basis2, raw2 = _solve_tableau(M, vrow0, vcol0)
                    assert ok2 and basis2 == basis, (jm, cur, rng_, mid)
                    assert _rel(-sigma * raw2 - result, slope * (mid - cur), 1e-9 * max(1.0, abs(result))), (jm, cur, mid)
                M = M0.copy()
                apply(M, end + out * 1e-3 * (width if width else max(1.0, abs(end - cur))))
                ok3, basis3, _ = _solve_tableau(M, vrow0, vcol0)
                assert not ok3 or basis3 != basis, (jm, cur, rng_, end)
        lps += 1
    assert ends >= 100, ends


def test_berlin_airlift_known_answers():
    """max 20000 brit + 30000 yank  s.t.  plane: b + y <= 44,  person: 8b + 16y <= 512,  cost: 5b + 9y <= 300,
    yankees: -2b + y = 0 (two rows: `min` first, then `max`).

    With y = 2b the binding row is person: 40b = 512, so b = 12.8, y = 25.6, result = 80000 b = 1 024 000.
    plane uses 38.4 (slack 5.6), cost uses 294.4 (slack 5.6).  The yankees rows leave one slack basic at 0; the other
    is non-basic.  Which one: raising the `min` row's slack e gives -2b + y = e, b = (512 - 16e)/40, y = 2b + e, so
    d result / d e = -0.4 * 20000 + 0.2 * 30000 = -2000 <= 0 (optimal), while the `max` row's slack moves the other way
    (+2000, not optimal).  So the `max` row's slack is basic and the `min` row's is non-basic.

    Duals: person p: b = p/40, result = 2000 p, dual 2000.  yankees t (the `min` row): b = (512 - 16t)/40,
    result = 1 024 000 - 2000 t, dual -2000; the `max` row's dual is 0 and so are plane's and cost's.
    RHS ranges: person keeps b, y >= 0 for p >= 0, plane 3p/40 <= 44 and cost 23p/40 <= 300: [0, 12000/23].  The
    yankees `min` row: t <= 0 keeps the basic `max` slack (= -t) >= 0, and plane (1536 - 8t)/40 <= 44 and cost
    (11776 - 8t)/40 <= 300 both give t >= -28: [-28, 0].  Its `max` row (slack basic at 0): [0, +inf).
    plane: [44 - 5.6, +inf) = [38.4, +inf); cost: [294.4, +inf).
    Cost ranges keep both non-basic reduced costs <= 0: person slack -(c_b + 2 c_y)/40 <= 0 and yankees slack
    -0.4 c_b + 0.2 c_y <= 0.  brit (c_y = 30000): c_b >= -60000 and c_b >= 15000: [15000, +inf).
    yank (c_b = 20000): c_y >= -10000 and c_y <= 40000: [-10000, 40000]."""
    from oracle import ref_model
    from oracle import sensitivity as S
    jm = _fixture("Berlin Air Lift Problem.json")
    rep = S.report(jm, ref_model.solve_full(jm))
    inf = float("inf")
    want = [("plane", "max", 5.6, 0.0, 38.4, inf), ("person", "max", 0.0, 2000.0, 0.0, 12000 / 23),
            ("cost", "max", 5.6, 0.0, 294.4, inf), ("yankees", "min", 0.0, -2000.0, -28.0, 0.0),
            ("yankees", "max", 0.0, 0.0, 0.0, inf)]
    assert len(rep["constraints"]) == len(want)
    close = lambda a, b: a == b or abs(a - b) <= 1e-12 * max(1.0, abs(b))
    for got, (name, kind, slack, dual, lo, hi) in zip(rep["constraints"], want):
        assert (got["name"], got["type"]) == (name, kind)
        assert close(got["slack"], slack) and close(got["dual"], dual), got
        assert close(got["range"]["min"], lo) and close(got["range"]["max"], hi), got
    assert {k: round(v, 6) for k, v in rep["duals"].items()} == {"plane": 0.0, "person": 2000.0, "cost": 0.0, "yankees": -2000.0}
    b, y = rep["variables"]["brit"], rep["variables"]["yank"]
    assert close(b["value"], 12.8) and close(y["value"], 25.6) and b["reducedCost"] == y["reducedCost"] == 0.0
    assert close(b["range"]["min"], 15000.0) and b["range"]["max"] == inf
    assert close(y["range"]["min"], -10000.0) and close(y["range"]["max"], 40000.0)
    assert not b["fixed"] and not y["fixed"]


class _StubTableau:
    """Stands in for GpuTableau: serves the oracle's final tableau through the two read-backs the report makes."""

    def __init__(self, model, sol=None):
        self.model = model
        self.handle = None
        self._version, self._solved_version = 0, -1
        if sol is not None:
            from oracle import sensitivity as S
            self.handle = object()
            self._solved_version = 0
            M = sol.tableau.matrix()
            vr, vc = sol.tableau.maps()
            unres = np.zeros(M.shape[0] + M.shape[1] - 2, dtype=np.uint8)
            for i in sol.model.unrestrictedVariables:
                unres[i] = 1
            self._state = (M[:, 0].copy(), M[0].copy(), vr, vc)
            self._bounds = S.bounds(M, vr, vc, unres, sol.model.precision)

    def final_state(self):
        return self._state

    def sensitivity_bounds(self):
        return self._bounds


def _cpu_model(jm, monkeypatch):
    import jslpsolver_b200.tableau as T
    from jslpsolver_b200.model import Model, presolve
    monkeypatch.setattr(T, "GpuTableau", lambda *a, **k: None)
    m = Model().loadJson(jm)
    m.presolveResult = presolve(m)
    for v in m.presolveResult.fixedVariables:
        v.cost = 0
    return m


def _soft(jm):
    return any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())


@pytest.mark.parametrize("fx", [f for f in BUNDLE["fixtures"] + BUNDLE["readme"]
                                if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"]))
                                and isinstance(f["model"].get("optimize"), str)],
                         ids=lambda f: f["file"])
def test_host_report_matches_the_restatement(fx, monkeypatch):
    """Solution.sensitivity()'s host assembly (names, signs, fixed variables, unrestricted columns) over the oracle's
    final tableau equals the oracle's own report, value for value."""
    from jslpsolver_b200.tableau import Solution
    from oracle import ref_model
    from oracle import sensitivity as S
    jm = strip_timeouts(fx["model"])
    sol = ref_model.solve_full(jm, fast_cycles=True)
    if sol.tableau is None or not (sol.feasible and sol.bounded):
        pytest.skip("no optimum")
    m = _cpu_model(jm, monkeypatch)
    t = _StubTableau(m, sol)
    assert Solution(t, sol.evaluation, True, True).sensitivity() == S.report(jm, sol)


def test_value_errors(monkeypatch):
    """Integer or binary variables, soft constraints, an infeasible or unbounded result, a tableau never solved or
    edited since the solve: each raises ValueError before anything is read from the device."""
    from jslpsolver_b200.tableau import Solution
    lp = _fixture("Berlin Air Lift Problem.json")
    cases = [
        (_fixture("Integer Berlin Air Lift Problem.json"), True, True, "integer or binary"),
        (dict(lp, binaries={"brit": 1}), True, True, "integer or binary"),
        (dict(lp, constraints=dict(lp["constraints"], plane={"max": 44, "weight": 10})), True, True, "soft constraints"),
        (dict(lp, constraints=dict(lp["constraints"], plane={"max": 44, "priority": "strong"})), True, True, "soft constraints"),
        (lp, False, True, "infeasible"),
        (lp, True, False, "unbounded"),
        (lp, True, True, "has not been solved"),
    ]
    for jm, feasible, bounded, match in cases:
        t = _StubTableau(_cpu_model(jm, monkeypatch))
        with pytest.raises(ValueError, match=match):
            Solution(t, 0.0, feasible, bounded).sensitivity()
    # solved, then edited (or solved again) after the Solution was made
    from oracle import ref_model
    t = _StubTableau(_cpu_model(lp, monkeypatch), ref_model.solve_full(lp))
    s = Solution(t, 0.0, True, True)
    s.sensitivity()
    t._version += 1
    with pytest.raises(ValueError, match="edited or solved again"):
        s.sensitivity()
    with pytest.raises(ValueError, match="needs a solution of a Model"):
        Solution(_StubTableau(None), 0.0, True, True).sensitivity()


def test_ctypes_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+jslp_sensitivity\s*\(([^)]*)\)\s*;", header)
    assert proto, "jslp_sensitivity is not declared"
    params = [p.strip() for p in proto.group(1).split(",")]
    assert [re.sub(r"\s+", " ", p.rsplit("*", 1)[0]).strip() + " *" for p in params] == \
        ["jslp_tab *", "double *", "double *", "double *", "double *"], params
    (name, res, args), = [s for s in _lib.SYMBOLS if s[0] == "jslp_sensitivity"]
    assert res is _lib.C.c_int and len(args) == len(params) and all(a is _lib.C.c_void_p for a in args)

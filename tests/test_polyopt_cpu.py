"""Polyopt and model validation on the host: the known answers of the reference's polyopt.test.ts and
validation.test.ts, and Polyopt over the oracle's Solve checked against SciPy HiGHS."""
import copy
import random
import warnings

import numpy as np
import pytest

from jslpsolver_b200 import validation
from jslpsolver_b200.polyopt import Polyopt

from helpers import highs_solve


class MockSolver:
    """createMockSolver (polyopt.test.ts:8-17): returns the listed solutions in turn, the last one repeated."""

    def __init__(self, solutions):
        self.solutions, self.calls = solutions, []

    def Solve(self, model, precision=None, full=None, validate=None):
        self.calls.append((copy.deepcopy(model), precision, full, validate))
        sol = self.solutions[min(len(self.calls) - 1, len(self.solutions) - 1)]
        return copy.deepcopy(sol) if isinstance(sol, dict) else sol


def two(obj1="max", obj2="max"):
    return {"optimize": {"obj1": obj1, "obj2": obj2}, "opType": "max", "constraints": {},
            "variables": {"x": {"obj1": 10, "obj2": 5}}}


@pytest.fixture
def mock():
    return MockSolver


def test_empty_objectives_raise(mock):
    with pytest.raises(ValueError, match="Multi-objective solve requires at least one objective definition"):
        Polyopt(mock([{}]), {"optimize": {}, "opType": "max", "constraints": {}, "variables": {}})


def test_single_and_multi_objective(mock):
    r = Polyopt(mock([{"feasible": True, "result": 10, "x": 5, "profit": 10}] * 2),
                {"optimize": {"profit": "max"}, "opType": "max", "constraints": {}, "variables": {"x": {"profit": 2}}})
    assert len(r["vertices"]) == 1 and set(r) == {"midpoint", "vertices", "ranges"}
    r = Polyopt(mock([{"feasible": True, "result": 100, "x": 10, "profit": 100, "efficiency": 0.5},
                      {"feasible": True, "result": 0.9, "x": 5, "profit": 50, "efficiency": 0.9},
                      {"feasible": True, "result": 75, "x": 7.5, "profit": 75, "efficiency": 0.7}]),
                {"optimize": {"profit": "max", "efficiency": "max"}, "opType": "max", "constraints": {},
                 "variables": {"x": {"profit": 10, "efficiency": 0.1}}})
    assert len(r["vertices"]) == 2 and r["midpoint"]["result"] == 75


def test_unique_and_duplicate_vertices(mock):
    r = Polyopt(mock([{"feasible": True, "result": 100, "x": 10, "obj1": 100, "obj2": 50},
                      {"feasible": True, "result": 80, "x": 8, "obj1": 80, "obj2": 80},
                      {"feasible": True, "result": 90, "x": 9}]), two())
    assert len(r["vertices"]) == 2
    s = mock([{"feasible": True, "result": 100, "x": 10, "obj1": 100, "obj2": 50},
              {"feasible": True, "result": 100, "x": 10, "obj1": 100, "obj2": 50},
              {"feasible": True, "result": 100, "x": 10}])
    r = Polyopt(s, two())
    assert len(r["vertices"]) == 1
    # the midpoint rows average over the unique vertices only; backfill adds x's contribution (10 * 10, 10 * 5) on
    # top of the value the solver reported, as polyopt.ts:64-74 does
    assert s.calls[-1][0]["constraints"] == {"obj1": {"equal": 200.0}, "obj2": {"equal": 100.0}}


def test_metadata_stripped(mock):
    r = Polyopt(mock([{"feasible": True, "result": 100, "bounded": True, "x": 10, "profit": 100},
                      {"feasible": True, "result": 100, "x": 10, "profit": 100}]),
                {"optimize": {"profit": "max"}, "opType": "max", "constraints": {}, "variables": {"x": {"profit": 10}}})
    assert not {"feasible", "result", "bounded"} & set(r["vertices"][0])


def test_ranges(mock):
    r = Polyopt(mock([{"feasible": True, "result": 100, "obj1": 100, "obj2": 20},
                      {"feasible": True, "result": 80, "obj1": 50, "obj2": 80},
                      {"feasible": True, "result": 90}]), two())
    assert r["ranges"]["obj1"] == {"min": 50, "max": 100} and r["ranges"]["obj2"] == {"min": 20, "max": 80}


def test_ranges_fill_missing_with_zero(mock):
    # backfill gives obj2 = 0 * 5 for the first vertex (x is absent): the implicit zero counts
    r = Polyopt(mock([{"feasible": True, "result": 100, "obj1": 100},
                      {"feasible": True, "result": 80, "obj1": 50, "obj2": 80},
                      {"feasible": True, "result": 90}]), two())
    assert r["ranges"]["obj2"]["min"] == 0


def test_backfill(mock):
    r = Polyopt(mock([{"feasible": True, "result": 50, "x": 5, "y": 3}] * 2),
                {"optimize": {"profit": "max"}, "opType": "max", "constraints": {},
                 "variables": {"x": {"profit": 10}, "y": {"profit": 5}}})
    assert r["vertices"][0]["profit"] == 65
    r = Polyopt(mock([{"feasible": True, "result": 100, "profit": 100}] * 2),
                {"optimize": {"profit": "max"}, "opType": "max", "constraints": {}, "variables": {"profit": {"cost": 1}}})
    assert r["vertices"][0]["profit"] == 100


def test_solver_interaction(mock):
    s = mock([{"feasible": True, "result": 100, "obj1": 100, "obj2": 50},
              {"feasible": True, "result": 80, "obj1": 50, "obj2": 80},
              {"feasible": True, "result": 75, "obj1": 75, "obj2": 65}])
    Polyopt(s, two())
    assert len(s.calls) == 3
    assert all(c[1:] == (None, None, True) for c in s.calls)


def test_caller_model_unchanged(mock):
    model = {"optimize": {"profit": "max"}, "opType": "max", "constraints": {"time": {"max": 100}},
             "variables": {"x": {"profit": 10, "time": 2}}}
    before = copy.deepcopy(model)
    Polyopt(mock([{"feasible": True, "result": 100, "profit": 100}] * 2), model)
    assert model == before


@pytest.mark.parametrize("bad", ["not an object", None])
def test_non_object_result_raises(mock, bad):
    with pytest.raises(ValueError, match="Polyopt requires the solver to return an object result"):
        Polyopt(mock([bad]), {"optimize": {"profit": "max"}, "opType": "max", "constraints": {},
                              "variables": {"x": {"profit": 10}}})


def test_midpoint_model(mock, monkeypatch):
    monkeypatch.setattr(random, "random", lambda: 0.25)
    s = mock([{"feasible": True, "result": 75, "obj1": 75, "obj2": 65}])
    Polyopt(s, two())
    mid = s.calls[-1][0]
    assert mid["constraints"]["obj1"] == {"equal": 75.0} and "obj2" in mid["constraints"]
    assert mid["optimize"] == "cheater-0.25" and mid["opType"] == "max"
    assert mid["variables"]["x"]["cheater-0.25"] == 1


# ---- validation.test.ts -------------------------------------------------------------------------------------

@pytest.fixture
def fixed_random(monkeypatch):
    monkeypatch.setattr(random, "random", lambda: 0.123456789)


def test_clean_no_conflict(fixed_random):
    model = {"optimize": "profit", "opType": "max", "constraints": {"time": {"max": 100}, "budget": {"max": 500}},
             "variables": {"x": {"profit": 10, "time": 2, "budget": 5}, "y": {"profit": 15, "time": 3, "budget": 8}}}
    assert validation.CleanObjectiveAttributes(model) is model
    assert "profit" not in model["constraints"] and "time" in model["constraints"]


def test_clean_renames_conflict(fixed_random):
    model = {"optimize": "value", "opType": "max", "constraints": {"value": {"max": 100}, "other": {"min": 10}},
             "variables": {"x": {"value": 5, "other": 2}, "y": {"value": 8, "other": 3}}}
    r = validation.CleanObjectiveAttributes(model)
    assert "value" not in r["constraints"]
    assert r["constraints"]["0.123456789"] == {"max": 100} and r["constraints"]["other"] == {"min": 10}
    assert list(r["constraints"]) == ["other", "0.123456789"]  # deleted and re-inserted: last
    assert r["variables"]["x"]["0.123456789"] == 5 and r["variables"]["y"]["0.123456789"] == 8


def test_clean_variables_without_attribute(fixed_random):
    for optimize in ("value", {"value": "max"}):
        model = {"optimize": optimize, "opType": "max", "constraints": {"value": {"max": 100}},
                 "variables": {"x": {"value": 5}, "y": {"other": 3}}}
        r = validation.CleanObjectiveAttributes(model)
        assert r["variables"]["x"]["0.123456789"] == 5 and "0.123456789" not in r["variables"]["y"]
        assert r["constraints"] == {"0.123456789": {"max": 100}}


def test_clean_multi_objective(fixed_random):
    model = {"optimize": {"profit": "max", "efficiency": "max"}, "opType": "max", "constraints": {"time": {"max": 100}},
             "variables": {"x": {"profit": 10, "efficiency": 0.9, "time": 2}}}
    assert validation.CleanObjectiveAttributes(model) is model and list(model["optimize"]) == ["profit", "efficiency"]
    model = {"optimize": {"profit": "max", "fixed": "max"}, "opType": "max",
             "constraints": {"fixed": "equal", "other": {"max": 50}}, "variables": {"x": {"profit": 10, "fixed": 5, "other": 2}}}
    r = validation.CleanObjectiveAttributes(model)
    assert r["optimize"] == {"profit": "max"}


def test_clean_multiple_conflicts(monkeypatch):
    draws = iter([0.1, 0.2])
    monkeypatch.setattr(random, "random", lambda: next(draws))
    model = {"optimize": {"a": "max", "b": "max"}, "opType": "max", "constraints": {"a": {"max": 100}, "b": {"min": 10}},
             "variables": {"x": {"a": 5, "b": 3}}}
    r = validation.CleanObjectiveAttributes(model)
    assert r["constraints"] == {"0.1": {"max": 100}, "0.2": {"min": 10}}
    assert r["variables"]["x"] == {"a": 5, "b": 3, "0.1": 5, "0.2": 3}


def test_clean_edge_cases(fixed_random):
    m = {"optimize": "profit", "opType": "max", "constraints": {}, "variables": {"x": {"profit": 10}}}
    assert validation.CleanObjectiveAttributes(m) is m
    m = {"optimize": "value", "opType": "max", "constraints": {"value": {"max": 100}}, "variables": {}}
    assert validation.CleanObjectiveAttributes(m)["constraints"] == {"0.123456789": {"max": 100}}
    m = {"optimize": {}, "opType": "max", "constraints": {"some": {"max": 100}}, "variables": {"x": {"some": 5}}}
    assert validation.CleanObjectiveAttributes(m) is m and m["constraints"] == {"some": {"max": 100}}


@pytest.mark.parametrize("model,text", [
    ({"optimize": "profit", "optype": "max", "constraints": {}, "variables": {}}, "'optype' but expected 'opType'"),
    ({"optimise": "profit", "opType": "max", "constraints": {}, "variables": {}}, "'optimise' but expected 'optimize'"),
    ({"optimize": "profit", "opType": "max", "constraint": {}, "variables": {}}, "'constraint' but expected 'constraints'"),
    ({"optimize": "profit", "opType": "max", "constraints": {}, "vars": {}}, "'vars' but expected 'variables'"),
    ({"optimize": "profit", "opType": "max", "constraints": {}, "variables": {"x": {"profit": 1}}, "int": {"x": 1}},
     "'int' but expected 'ints'"),
    ({"opType": "max", "constraints": {}, "variables": {}}, "missing 'optimize' property"),
    ({"optimize": "profit", "constraints": {}, "variables": {}}, "missing 'opType' property"),
    ({"optimize": "profit", "opType": "max", "constraints": {"budget": {"minimum": 100}}, "variables": {}},
     "Constraint 'budget' has 'minimum' but expected 'min'"),
    ({"optimize": "profit", "opType": "max", "constraints": {"capacity": {"maximum": 500}}, "variables": {}},
     "Constraint 'capacity' has 'maximum' but expected 'max'"),
    ({"optimize": "profit", "opType": "max", "constraints": {"fixed": {"equals": 100}}, "variables": {}},
     "Constraint 'fixed' has 'equals' but expected 'equal'"),
])
def test_warn_on_typos(model, text):
    with pytest.warns(UserWarning, match=text.replace("(", r"\(")) as rec:
        assert validation.WarnOnTypos(model) is model
    assert all(str(w.message).startswith("[jsLPSolver] Warning: ") for w in rec)


def test_warn_typo_suppresses_missing_optype():
    with pytest.warns(UserWarning) as rec:
        validation.WarnOnTypos({"optimize": "profit", "optype": "max", "constraints": {}, "variables": {}})
    texts = [str(w.message) for w in rec]
    assert any("'optype' but expected 'opType'" in t for t in texts)
    assert not any("missing 'opType'" in t for t in texts)


def test_valid_model_does_not_warn():
    model = {"optimize": "profit", "opType": "max", "constraints": {"budget": {"max": 100}, "time": {"min": 10}},
             "variables": {"x": {"profit": 10, "budget": 5, "time": 2}}, "ints": {"x": 1}}
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        assert validation.WarnOnTypos(model) is model


# ---- Polyopt over the oracle vs SciPy HiGHS -----------------------------------------------------------------

def random_multi_model(seed: int) -> dict:
    """Bounded, feasible LP: `max` packing rows over every variable (x = 0 is feasible), a few sparse `min` rows with
    small right-hand sides, and 2-4 objectives of either sense.  Every row has two or more variables: the reference's
    presolve drops a single-variable row and keeps its bound only when it fixes the variable (presolve.ts:343-467)."""
    rng = np.random.default_rng(seed)
    n, m, k = int(rng.integers(3, 9)), int(rng.integers(2, 7)), int(rng.integers(2, 5))
    variables = {f"x{j}": {} for j in range(n)}
    constraints = {}
    for i in range(m):
        for j in range(n):
            if i == 0 or j < 2 or rng.random() < 0.7:
                variables[f"x{j}"][f"r{i}"] = float(rng.integers(1, 21))
        constraints[f"r{i}"] = {"max": float(rng.integers(100, 501))}
    for i in range(int(rng.integers(0, 3))):
        for j in rng.choice(n, 2, replace=False):
            variables[f"x{j}"][f"q{i}"] = float(rng.integers(1, 5))
        constraints[f"q{i}"] = {"min": float(rng.integers(1, 10))}
    optimize = {}
    for o in range(k):
        for j in range(n):
            if rng.random() < 0.8:
                variables[f"x{j}"][f"o{o}"] = float(rng.integers(1, 51))
        optimize[f"o{o}"] = "max" if rng.random() < 0.7 else "min"
    return {"optimize": optimize, "opType": "max", "constraints": constraints, "variables": variables}


class OracleSolver:
    """Solve(model, precision, full, validate) over the oracle, recording each per-objective solution."""

    def __init__(self):
        from oracle import ref_model
        self.ref, self.per_objective, self.models = ref_model, {}, []

    def Solve(self, model, precision=None, full=None, validate=None):
        if validate:
            model = validation.validate(model)
        self.models.append(copy.deepcopy(model))
        sol = self.ref.Solve(model, precision, bool(full))
        self.per_objective.setdefault(model["optimize"], sol)
        return sol


@pytest.mark.parametrize("seed", range(30))
def test_polyopt_oracle_vs_highs(seed):
    model = random_multi_model(seed)
    s = OracleSolver()
    out = Polyopt(s, model)
    for name, sense in model["optimize"].items():
        sol = s.per_objective[name]
        assert sol["feasible"] and sol["bounded"]
        single = {"optimize": name, "opType": sense, "constraints": model["constraints"], "variables": model["variables"]}
        status, best = highs_solve(single)
        assert status == 0
        assert sol[name] == pytest.approx(best, rel=1e-7, abs=1e-9), name   # backfilled objective value
    mid_rows = s.models[-1]["constraints"]
    assert set(mid_rows) == set(model["constraints"]) | set(model["optimize"])
    assert 1 <= len(out["vertices"]) <= len(model["optimize"])

    def check_rows(x):
        for cname, spec in mid_rows.items():
            lhs = sum(coefs.get(cname, 0.0) * x[v] for v, coefs in model["variables"].items())
            tol = 1e-7 * max(1.0, max(abs(b) for b in spec.values()))
            if "equal" in spec:
                assert abs(lhs - spec["equal"]) <= tol, cname
            if "max" in spec:
                assert lhs <= spec["max"] + tol, cname
            if "min" in spec:
                assert lhs >= spec["min"] - tol, cname

    # the midpoint model always has a solution: the average of the vertices
    check_rows({v: float(np.mean([vx.get(v, 0.0) for vx in out["vertices"]])) for v in model["variables"]})
    mid = out["midpoint"]
    if seed == 11:  # vertices are rounded to 1e-8 before averaging: the reference's phase 1 rejects this midpoint
        assert not mid["feasible"]
        return
    assert mid["feasible"]
    check_rows({v: mid.get(v, 0.0) for v in model["variables"]})

"""Multi-objective Solve on the GPU against Polyopt driven by the oracle's Solve, bit for bit."""
import random
import struct
import warnings

import pytest

pytestmark = pytest.mark.gpu


class OracleSolver:
    def Solve(self, model, precision=None, full=None, validate=None):
        from jslpsolver_b200 import validation
        from oracle import ref_model
        if validate:
            model = validation.validate(model)
        return ref_model.Solve(model, precision, bool(full), fast_cycles=True)


def assert_same(a, b, path="result"):
    """Equal structure, key order and float bits."""
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b), (path, list(a), list(b))
        for k in a:
            assert_same(a[k], b[k], f"{path}.{k}")
    elif isinstance(a, list):
        assert isinstance(b, list) and len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, f"{path}[{i}]")
    elif isinstance(a, float) or isinstance(b, float):
        assert struct.pack("<d", float(a)) == struct.pack("<d", float(b)), (path, a, b)
    else:
        assert type(a) is type(b) and a == b, (path, a, b)


def polyopt_parity(model, solver=None, seed=7):
    import jslpsolver_b200 as J
    from jslpsolver_b200.polyopt import Polyopt
    solver = solver or J.Solver()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        random.seed(seed)
        got = solver.Solve(model)
        random.seed(seed)
        want = Polyopt(OracleSolver(), model)
    assert_same(got, want)
    return got


AIRLIFT = {"optimize": {"capacity": "max", "cost": "min"}, "opType": "max",
           "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
           "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                         "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}


def test_berlin_airlift_two_objectives():
    out = polyopt_parity(AIRLIFT)  # `cost` is also a constraint: validation renames it, moving that row last
    assert len(out["vertices"]) == 2 and out["midpoint"]["feasible"]


def test_objective_named_like_a_constraint_reorders_rows():
    model = {"optimize": {"a": "max", "b": "max"}, "opType": "max",
             "constraints": {"a": {"max": 40}, "c1": {"max": 30}, "b": {"max": 50}, "c2": {"max": 25}},
             "variables": {"x": {"a": 2, "b": 1, "c1": 1, "c2": 1}, "y": {"a": 1, "b": 3, "c1": 2},
                           "z": {"a": 1, "b": 1, "c2": 3}}}
    polyopt_parity(model)


def test_objective_named_like_a_variable_skips_backfill():
    model = {"optimize": {"x": "max", "profit": "max"}, "opType": "max",
             "constraints": {"cap": {"max": 10}, "mix": {"max": 14}},
             "variables": {"x": {"cap": 1, "mix": 2, "profit": 1}, "y": {"cap": 1, "mix": 1, "profit": 3}}}
    polyopt_parity(model)


def test_duplicate_vertices():
    model = {"optimize": {"p": "max", "q": "max"}, "opType": "max",
             "constraints": {"cap": {"max": 10}},
             "variables": {"x": {"cap": 1, "p": 3, "q": 6}, "y": {"cap": 1, "p": 1, "q": 2}}}
    assert len(polyopt_parity(model)["vertices"]) == 1


def test_mip_objectives():
    model = {"optimize": {"value": "max", "weight": "min"}, "opType": "max",
             "constraints": {"cap": {"max": 23}, "count": {"min": 2}},
             "variables": {f"i{j}": {"value": 3 + (7 * j) % 11, "weight": 2 + (5 * j) % 9, "cap": 2 + (5 * j) % 9,
                                     "count": 1} for j in range(8)},
             "ints": {f"i{j}": 1 for j in range(8)}}
    polyopt_parity(model)


def test_weight_priority_model():
    model = {"optimize": {"profit": "max", "quality": "max"}, "opType": "max",
             "constraints": {"cap": {"max": 20}, "want": {"min": 30, "weight": 2, "priority": "strong"}},
             "variables": {"x": {"cap": 2, "want": 3, "profit": 5, "quality": 1},
                           "y": {"cap": 1, "want": 1, "profit": 2, "quality": 4}}}
    polyopt_parity(model)


def test_resident_size_model():
    from jslpsolver_b200 import problems
    polyopt_parity(problems.dense_packing_multi_model(20, 15, 3, seed=5))


@pytest.mark.parametrize("n_obj,n,m", [(2, 160, 130), (3, 150, 140), (5, 140, 120), (3, 300, 250)])
def test_dense_packing_objectives(n_obj, n, m):
    from jslpsolver_b200 import problems
    polyopt_parity(problems.dense_packing_multi_model(n, m, n_obj, seed=n_obj))


def test_single_objective_validate_and_multi_objective_entry_points():
    import jslpsolver_b200 as J
    from oracle import ref_model
    model = {"optimize": "cost", "opType": "min", "constraints": {"cost": {"min": 3}, "cap": {"max": 10}},
             "variables": {"x": {"cost": 2, "cap": 1}, "y": {"cost": 3, "cap": 2}}}
    random.seed(1)
    got = J.Solve(dict(model, constraints=dict(model["constraints"])), None, False, True)
    random.seed(1)
    want = ref_model.Solve(J.validation.validate(dict(model, constraints=dict(model["constraints"]))))
    assert_same(got, want)
    random.seed(3)
    a = J.solver.MultiObjective(AIRLIFT)
    random.seed(3)
    assert_same(a, J.Solve(AIRLIFT))

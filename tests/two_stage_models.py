"""Two-stage stochastic LP fixtures (DESIGN.md section 2u) and the deterministic equivalent solved by SciPy HiGHS, shared
by the CPU and GPU tests of TwoStage()."""
from __future__ import annotations

import numpy as np

# Birge and Louveaux's farmer: 500 acres of wheat, corn and sugar beets planted now, yields known after planting (above
# average, average, below average, equally likely); the published plan is 170 / 80 / 250 acres, expected profit 108390.
FARMER = {"optimize": "profit", "opType": "max",
          "constraints": {"land": {"max": 500}, "wheat": {"min": 200}, "corn": {"min": 240}, "beets": {"max": 0},
                          "quota": {"max": 6000}},
          "variables": {"wheat_acres": {"profit": -150, "land": 1, "wheat": 2.5},
                        "corn_acres": {"profit": -230, "land": 1, "corn": 3},
                        "beet_acres": {"profit": -260, "land": 1, "beets": -20},
                        "wheat_bought": {"profit": -238, "wheat": 1}, "wheat_sold": {"profit": 170, "wheat": -1},
                        "corn_bought": {"profit": -210, "corn": 1}, "corn_sold": {"profit": 150, "corn": -1},
                        "beets_sold": {"profit": 36, "beets": 1, "quota": 1}, "beets_extra": {"profit": 10, "beets": 1}}}
FARMER_FIRST = ["wheat_acres", "corn_acres", "beet_acres"]
FARMER_CASES = [{"coefficients": {"wheat": {"wheat_acres": w}, "corn": {"corn_acres": c}, "beets": {"beet_acres": -b}}}
                for w, c, b in ((3.0, 3.6, 24), (2.5, 3.0, 20), (2.0, 2.4, 16))]


def capacity(seed: int, n_first=3, n_second=4, n_cases=5, per_case_t=False, complete=True, max_sense=False):
    """A seeded capacity-expansion model: build capacity x_i now (cost, budget row), then in each case serve demand d_k
    from the capacities (y_ik <= x_i links), unmet demand at a penalty when `complete` (otherwise a case whose demand
    exceeds what x can serve is infeasible, which needs feasibility cuts)."""
    rng = np.random.default_rng(seed)
    cons, var = {"budget": {"max": float(rng.integers(40, 80))}}, {}
    obj = "cost"
    sign = -1 if max_sense else 1
    for i in range(n_first):
        var[f"x{i}"] = {obj: sign * float(rng.integers(1, 6)), "budget": float(rng.integers(1, 4))}
    for k in range(n_second):
        cons[f"demand{k}"] = {"min": float(rng.integers(2, 10))}
    for i in range(n_first):
        cons[f"link{i}"] = {"max": 0.0}
        var[f"x{i}"][f"link{i}"] = -float(rng.integers(1, 3))
        for k in range(n_second):
            if rng.random() < 0.7 or i == k % n_first:
                var[f"y{i}_{k}"] = {obj: sign * float(rng.integers(1, 5)), f"demand{k}": 1.0, f"link{i}": 1.0}
    if complete:
        for k in range(n_second):
            var[f"short{k}"] = {obj: sign * 40.0, f"demand{k}": 1.0}
    cases = []
    for _ in range(n_cases):
        case = {"rhs": {f"demand{k}": float(rng.integers(1, 14)) for k in range(n_second) if rng.random() < 0.8}}
        if rng.random() < 0.5:
            ys = [v for v in var if v.startswith("y")]
            case["cost"] = {ys[int(rng.integers(len(ys)))]: sign * float(rng.integers(1, 6))}
        if per_case_t:
            case["coefficients"] = {f"link{i}": {f"x{i}": -float(rng.integers(1, 4))} for i in range(n_first)
                                    if rng.random() < 0.6}
        cases.append(case)
    model = {"optimize": obj, "opType": "max" if max_sense else "min", "constraints": cons, "variables": var}
    probabilities = [float(v) for v in rng.integers(1, 5, size=n_cases)]
    return model, cases, [f"x{i}" for i in range(n_first)], probabilities


def deterministic_equivalent(model, cases, first, probabilities=None):
    """linprog of the deterministic equivalent: (status, objective in the model's sense)."""
    from scipy.optimize import linprog
    obj, sense = model["optimize"], -1.0 if model.get("opType") == "max" else 1.0
    variables, constraints = model["variables"], model["constraints"]
    second = [v for v in variables if v not in first]
    srows = [n for n in constraints if any(variables[y].get(n, 0) for y in second)]
    frows = [n for n in constraints if n not in srows]
    n = len(cases)
    p = np.ones(n) / n if probabilities is None else np.asarray(probabilities, float) / sum(probabilities)
    nx, ny = len(first), len(second)
    cols = nx + n * ny
    c = np.zeros(cols)
    for j, x in enumerate(first):
        c[j] = sense * variables[x].get(obj, 0)
    A, b = [], []

    def add(row, spec_row, lo_hi):
        for side, v in lo_hi.items():
            if side == "max":
                A.append(row), b.append(v)
            elif side == "min":
                A.append(-row), b.append(-v)
            else:
                A.append(row), b.append(v), A.append(-row), b.append(-v)
    for nm in frows:
        row = np.zeros(cols)
        for j, x in enumerate(first):
            row[j] = variables[x].get(nm, 0)
        add(row, nm, {k: v for k, v in constraints[nm].items() if k in ("min", "max", "equal") and v is not None})
    for s, case in enumerate(cases):
        costs = case.get("cost") or {}
        for j, y in enumerate(second):
            c[nx + s * ny + j] = sense * p[s] * costs.get(y, variables[y].get(obj, 0))
        for nm in srows:
            row = np.zeros(cols)
            tech = (case.get("coefficients") or {}).get(nm, {})
            for j, x in enumerate(first):
                row[j] = tech.get(x, variables[x].get(nm, 0))
            for j, y in enumerate(second):
                row[nx + s * ny + j] = variables[y].get(nm, 0)
            spec = {k: v for k, v in constraints[nm].items() if k in ("min", "max", "equal") and v is not None}
            r = (case.get("rhs") or {}).get(nm)
            if isinstance(r, dict):
                spec.update(r)
            elif r is not None:
                spec = {k: r for k in spec}
            add(row, nm, spec)
    res = linprog(c, A_ub=np.array(A), b_ub=np.array(b), bounds=[(0, None)] * cols, method="highs")
    return res.status, (sense * res.fun if res.status == 0 else None)

"""The Pareto frontier of a two-objective MIP (DESIGN.md section 2s) without a GPU: the restatement of
tests/frontier_mip_oracle.py against brute-force enumeration of every plan of tiny binary models (the three-point
example's unsupported point included) and against an independent epsilon-constraint loop of sequential lexmins over
SciPy's HiGHS `milp` on seeded two-objective knapsacks, assignment and set-cover models and planted models with
unsupported points; the properties of the answer (nondominated, frontier order, ends equal to LexicographicMIP() in
both key orders, a too-large step reported through `exact`); every stop and every refusal; and the jslp_box_batch
declaration against its ctypes mirror."""
from __future__ import annotations

import itertools

import numpy as np
import pytest

import frontier_mip_oracle as FO
import lexicographic_mip_oracle as LMO
from jslpsolver_b200.frontier import _coef
from jslpsolver_b200.model import object_keys
from test_mip_variability_cpu import lp_data
from test_pool_cpu import _types

TOL = 1e-6

# binaries x, y, z with x + y + z = 1; min g1 = 3y + 4z, min g2 = 4x + 3y: (3, 3) is above the line through the ends
EXAMPLE = {"optimize": {"g1": "min", "g2": "min"}, "constraints": {"one": {"equal": 1}},
           "variables": {"x": {"one": 1, "g2": 4}, "y": {"one": 1, "g1": 3, "g2": 3}, "z": {"one": 1, "g1": 4}},
           "binaries": {"x": 1, "y": 1, "z": 1}}


@pytest.fixture(scope="module", autouse=True)
def _oracle_lib():
    from oracle import ref_model
    ref_model.build_oracle()


# ---- families -----------------------------------------------------------------------------------------------------
def knapsack(n: int, seed: int) -> dict:
    """Bi-objective 0/1 knapsack: max p1, max p2 under one weight row of half the total weight."""
    rng = np.random.default_rng(seed)
    w, p1, p2 = (rng.integers(1, 30, size=n) for _ in range(3))
    return {"name": f"knapsack{n}-{seed}", "optimize": {"p1": "max", "p2": "max"},
            "constraints": {"weight": {"max": int(w.sum()) // 2}},
            "variables": {f"x{j}": {"weight": int(w[j]), "p1": int(p1[j]), "p2": int(p2[j])} for j in range(n)},
            "binaries": {f"x{j}": 1 for j in range(n)}}


def assignment(n: int, seed: int) -> dict:
    """n x n assignment with two cost matrices, both minimised."""
    rng = np.random.default_rng(seed)
    c1, c2 = rng.integers(1, 20, size=(n, n)), rng.integers(1, 20, size=(n, n))
    variables = {f"a{i}_{j}": {f"r{i}": 1, f"c{j}": 1, "cost": int(c1[i, j]), "time": int(c2[i, j])}
                 for i in range(n) for j in range(n)}
    cons = {**{f"r{i}": {"equal": 1} for i in range(n)}, **{f"c{j}": {"equal": 1} for j in range(n)}}
    return {"name": f"assignment{n}-{seed}", "optimize": {"cost": "min", "time": "min"}, "constraints": cons,
            "variables": variables, "binaries": {v: 1 for v in variables}}


def set_cover(m: int, n: int, seed: int) -> dict:
    """Set cover of m elements by n random sets (every element in two at least), two costs minimised."""
    rng = np.random.default_rng(seed)
    member = rng.random((m, n)) < 0.35
    for e in range(m):
        member[e, rng.choice(n, size=2, replace=False)] = True
    variables = {f"s{j}": {**{f"e{e}": 1 for e in range(m) if member[e, j]}, "cost": int(rng.integers(1, 15)),
                           "risk": int(rng.integers(1, 15))} for j in range(n)}
    return {"name": f"cover{m}x{n}-{seed}", "optimize": {"cost": "min", "risk": "min"},
            "constraints": {f"e{e}": {"min": 1} for e in range(m)}, "variables": variables,
            "binaries": {v: 1 for v in variables}}


def planted(k: int, groups: int = 1) -> dict:
    """Pick one of k options per group: option i has g1 = 4i and g2 = 4(k-1-i), plus 3 on g2 for the interior ones,
    so every interior image lies above the line through the ends (unsupported)."""
    variables, cons = {}, {}
    for g in range(groups):
        cons[f"pick{g}"] = {"equal": 1}
        for i in range(k):
            variables[f"o{g}_{i}"] = {f"pick{g}": 1, "f1": 4 * i + g, "f2": 4 * (k - 1 - i) + (3 if 0 < i < k - 1 else 0)}
    return {"name": f"planted{k}x{groups}", "optimize": {"f1": "min", "f2": "min"}, "constraints": cons,
            "variables": variables, "binaries": {v: 1 for v in variables}}


def general_ints(seed: int) -> dict:
    """Two general integer variables under two rows, max f1 and min f2."""
    rng = np.random.default_rng(seed)
    return {"name": f"ints-{seed}", "optimize": {"f1": "max", "f2": "min"},
            "constraints": {"a": {"max": int(rng.integers(10, 20))}, "b": {"max": int(rng.integers(10, 20))}},
            "variables": {"x": {"a": int(rng.integers(1, 4)), "b": 1, "f1": int(rng.integers(1, 6)),
                                "f2": -int(rng.integers(0, 3))},
                          "y": {"a": 1, "b": int(rng.integers(1, 4)), "f1": int(rng.integers(1, 6)),
                                "f2": int(rng.integers(1, 6))}},
            "ints": {"x": 1, "y": 1}}


FAMILIES = ([knapsack(n, s) for n, s in ((6, 1), (8, 2), (10, 3))] + [assignment(3, 1), assignment(4, 2)] +
            [set_cover(6, 8, 1), set_cover(8, 10, 2)] + [planted(4), planted(6), planted(4, 2)] +
            [general_ints(s) for s in (1, 2)])


# ---- independent answers ------------------------------------------------------------------------------------------
def signs(jm):
    keys = object_keys(jm["optimize"])
    return keys, [1.0 if jm["optimize"][k] == "min" else -1.0 for k in keys]


def images(points, jm) -> list:
    keys, sig = signs(jm)
    return [tuple(s * p["objectives"][k] for k, s in zip(keys, sig)) for p in points]


def nondominated(imgs) -> list:
    imgs = sorted(set(imgs))
    return [p for p in imgs if not any(q[0] <= p[0] and q[1] <= p[1] and q != p for q in imgs)]


def brute_force(jm: dict) -> list:
    """The nondominated images (g1, g2) over every 0/1 plan of a binary model."""
    m, _, rows, _ = lp_data(dict(jm, optimize=object_keys(jm["optimize"])[0]))
    keys, sig = signs(jm)
    c = [np.array([s * _coef(jm, v.id, k) for v in m.variables]) for k, s in zip(keys, sig)]
    imgs = []
    for x in itertools.product((0.0, 1.0), repeat=len(m.variables)):
        x = np.array(x)
        if all((a @ x <= con.rhs + 1e-9) if con.isUpperBound else (a @ x >= con.rhs - 1e-9) for con, a in rows):
            imgs.append((float(c[0] @ x), float(c[1] @ x)))
    return nondominated(imgs)


def highs_frontier(jm: dict, step: float = 1.0) -> list:
    """The epsilon-constraint loop over HiGHS: from eps = inf, c = lexmin(g1, g2) under g2 <= eps, then eps = c2 - step,
    until no plan."""
    from scipy.optimize import Bounds, LinearConstraint, milp
    m, _, rows, integrality = lp_data(dict(jm, optimize=object_keys(jm["optimize"])[0]))
    keys, sig = signs(jm)
    c = [np.array([s * _coef(jm, v.id, k) for v in m.variables]) for k, s in zip(keys, sig)]
    A = np.array([a for _, a in rows])
    lo = np.array([-np.inf if con.isUpperBound else con.rhs for con, _ in rows])
    hi = np.array([con.rhs if con.isUpperBound else np.inf for con, _ in rows])
    out, eps = [], np.inf

    def solve(obj, extra):
        cons = [LinearConstraint(A, lo, hi)] + [LinearConstraint(row[None, :], -np.inf, u) for row, u in extra]
        r = milp(obj, constraints=cons, integrality=integrality, bounds=Bounds(0, np.inf),
                 options={"mip_rel_gap": 0, "presolve": True})
        return None if r.status != 0 else r.x

    while True:
        x = solve(c[0], [(c[1], eps)])
        if x is None:
            return out
        v1 = float(c[0] @ x)
        x = solve(c[1], [(c[1], eps), (c[0], v1 + 1e-6)])
        img = (float(c[0] @ x), float(c[1] @ x))
        out.append(img)
        eps = img[1] - step + 1e-6


def assert_close(got, want, what):
    assert len(got) == len(want), (what, got, want)
    for p, q in zip(got, want):
        assert abs(p[0] - q[0]) <= TOL and abs(p[1] - q[1]) <= TOL, (what, got, want)


# ---- against brute force and HiGHS -----------------------------------------------------------------------------------
def test_the_example_has_its_unsupported_point():
    out, _ = FO.frontier_mip(EXAMPLE)
    assert out["stop"] == "reached" and out["exact"] and out["open"] == []
    assert [(p["objectives"]["g1"], p["objectives"]["g2"]) for p in out["points"]] == [(0, 4), (3, 3), (4, 0)]
    assert [p["values"] for p in out["points"]][1] == {"x": 0.0, "y": 1.0, "z": 0.0}


@pytest.mark.parametrize("jm", [EXAMPLE, planted(4), planted(5, 2), knapsack(6, 4), knapsack(7, 5), assignment(3, 3),
                                set_cover(5, 7, 3)], ids=lambda m: m.get("name", "example"))
def test_equals_brute_force(jm):
    out, _ = FO.frontier_mip(jm, width=4)
    assert_close(images(out["points"], jm), brute_force(jm), jm.get("name"))
    assert out["exact"]


@pytest.mark.parametrize("jm", FAMILIES, ids=lambda m: m["name"])
def test_equals_the_epsilon_constraint_loop(jm):
    out, det = FO.frontier_mip(jm)
    assert out["stop"] == "reached" and out["exact"]
    assert_close(images(out["points"], jm), highs_frontier(jm), jm["name"])
    assert out["searches"] >= 2 and all(n >= 1 for n in det["stages"])


def test_planted_unsupported_points_are_found():
    jm = planted(6)
    out, _ = FO.frontier_mip(jm)
    imgs = images(out["points"], jm)
    assert len(imgs) == 6
    a, b = imgs[0], imgs[-1]
    for p in imgs[1:-1]:  # above the line through the ends: no weighted sum selects it
        assert (p[0] - a[0]) * (b[1] - a[1]) - (p[1] - a[1]) * (b[0] - a[0]) < 0


# ---- properties -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("jm", FAMILIES[:8], ids=lambda m: m["name"])
def test_properties(jm):
    out, _ = FO.frontier_mip(jm, width=16)
    imgs = images(out["points"], jm)
    assert imgs == sorted(imgs) and all(p[1] > q[1] for p, q in zip(imgs, imgs[1:])), "frontier order"
    assert imgs == nondominated(imgs), "a point is dominated by another"
    keys = object_keys(jm["optimize"])
    for order, end in ((keys, out["points"][0]), (keys[::-1], out["points"][-1])):
        lex, _ = LMO.chain(dict(jm, optimize={k: jm["optimize"][k] for k in order}))
        # the same plan; the frontier reports integer variables at their integers
        assert {k: round(x) for k, x in lex["values"].items()} == end["values"]
        assert all(abs(lex["objectives"][k] - end["objectives"][k]) <= TOL for k in keys)


def test_width_changes_no_point():
    jm = knapsack(8, 2)
    runs = [FO.frontier_mip(jm, width=w)[0] for w in (1, 3, 16)]
    for r in runs[1:]:
        assert images(r["points"], jm) == images(runs[0]["points"], jm)


def test_a_step_beyond_the_separation_drops_points_and_says_so():
    jm = planted(6)  # separation 4 in g1
    full, _ = FO.frontier_mip(jm)
    coarse, _ = FO.frontier_mip(jm, step=5)
    assert len(coarse["points"]) < len(full["points"]) and not coarse["exact"] and coarse["stop"] == "reached"
    fine, _ = FO.frontier_mip(jm, step=0.5)  # every coefficient a multiple of 0.5: still proven
    assert fine["exact"] and images(fine["points"], jm) == images(full["points"], jm)


def test_non_integer_coefficients_need_a_step():
    jm = {**EXAMPLE, "variables": {**EXAMPLE["variables"], "y": {"one": 1, "g1": 2.5, "g2": 3}}}
    with pytest.raises(ValueError, match="step= must be given"):
        FO.frontier_mip(jm)
    out, _ = FO.frontier_mip(jm, step=0.5)
    assert out["exact"] and [p["objectives"]["g1"] for p in out["points"]] == [0.0, 2.5, 4.0]
    out, _ = FO.frontier_mip(jm, step=0.3)
    assert not out["exact"] and len(out["points"]) == 3


# ---- stops ----------------------------------------------------------------------------------------------------------
def test_no_integer_plan():
    jm = {"optimize": {"a": "max", "b": "min"}, "constraints": {"odd": {"equal": 3}},
          "variables": {"x": {"odd": 2, "a": 1, "b": 1}, "y": {"odd": 2, "a": 1}}, "ints": {"x": 1, "y": 1}}
    out, _ = FO.frontier_mip(jm)
    assert not out["feasible"] and out["stop"] is None and out["points"] == [] and out["open"] == []


def test_one_point_frontier():
    jm = {"optimize": {"a": "max", "b": "max"}, "constraints": {"c": {"max": 3}},
          "variables": {"x": {"c": 1, "a": 1, "b": 2}}, "ints": {"x": 1}}
    out, _ = FO.frontier_mip(jm)
    assert out["stop"] == "reached" and out["exact"] and [p["values"] for p in out["points"]] == [{"x": 3.0}]


def test_an_unbounded_extreme_reports_the_other():
    jm = {"optimize": {"a": "max", "b": "min"}, "constraints": {"c": {"min": 1}},
          "variables": {"x": {"c": 1, "a": 1, "b": 1}, "y": {"c": 1, "a": 0, "b": 2}}, "ints": {"x": 1, "y": 1}}
    out, _ = FO.frontier_mip(jm)
    assert out["stop"] == "unbounded" and not out["bounded"] and not out["exact"]
    assert [p["objectives"] for p in out["points"]] == [{"a": 1.0, "b": 1.0}]


def test_max_points_leaves_open_boxes():
    jm = planted(8)
    out, _ = FO.frontier_mip(jm, max_points=4)
    assert out["stop"] == "limit" and not out["exact"] and out["open"]
    assert 2 <= len(out["points"]) <= 4
    full = images(FO.frontier_mip(jm)[0]["points"], jm)
    assert set(images(out["points"], jm)) <= set(full)
    for box in out["open"]:  # every open box lies between two reported points
        assert box["from"] in [p["objectives"] for p in out["points"]]
        assert box["to"] in [p["objectives"] for p in out["points"]]


@pytest.mark.parametrize("jm, max_nodes", [(knapsack(12, 7), 40), (planted(8), 5)], ids=["knapsack", "planted"])
def test_max_nodes_leaves_open_boxes(jm, max_nodes):
    out, _ = FO.frontier_mip(jm, max_nodes=max_nodes, width=1)
    assert out["stop"] == "limit" and not out["exact"] and out["open"]
    full = images(FO.frontier_mip(jm)[0]["points"], jm)
    assert set(images(out["points"], jm)) <= set(full)


def test_an_extreme_without_a_plan_at_max_nodes_is_refused():
    with pytest.raises(ValueError, match=r"the search for the optimum of 'p2' hit max_nodes=10 before any integer"):
        FO.frontier_mip(knapsack(12, 7), max_nodes=10, width=1)


def test_a_constraint_named_like_an_objective_keeps_the_box_rows_apart():
    """A budget row named `cost` beside the objective `cost`: the box rows live under fresh names, so the budget row
    is read as LexicographicMIP() reads it."""
    jm = {"optimize": {"profit": "max", "cost": "min"},
          "constraints": {"cost": {"max": 10}, "cap": {"max": 3}, "frontier.0": {"max": 100}},
          "variables": {f"x{j}": {"cap": 1, "profit": p, "cost": c, "frontier.0": 1}
                        for j, (p, c) in enumerate(((5, 4), (4, 2), (3, 1), (2, 1)))},
          "binaries": {f"x{j}": 1 for j in range(4)}}
    out, _ = FO.frontier_mip(jm)
    lex, _ = LMO.chain(jm)
    assert out["points"][0]["values"] == {k: round(x) for k, x in lex["values"].items()}
    assert_close(images(out["points"], jm), brute_force(dict(jm, optimize={"profit": "max", "cost": "min"})), "budget")


# ---- refusals -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model, kw, match", [
    ({**EXAMPLE, "binaries": {}}, {}, r"needs integer or binary variables: for a continuous LP use Frontier\(\)"),
    ({**EXAMPLE, "constraints": {"one": {"equal": 1, "weight": 2}}}, {}, "soft constraints"),
    ({**EXAMPLE, "unrestricted": {"x": 1}}, {}, "unrestricted variables"),
    ({**EXAMPLE, "external": {"solver": "lpsolve"}}, {}, "external solvers"),
    ({**EXAMPLE, "optimize": {"g1": "min"}}, {}, "exactly two objectives"),
    ({**EXAMPLE, "optimize": {"g1": "min", "g2": "min", "one": "max"}}, {}, "exactly two objectives"),
    ({**EXAMPLE, "variables": {**EXAMPLE["variables"], "w": {"one": 1, "g1": 1}}}, {},
     r"continuous variable 'w'; with continuous variables in an objective the frontier has segments"),
    (EXAMPLE, {"step": 0}, "step= must be a finite number > 0"),
    (EXAMPLE, {"step": float("inf")}, "step= must be a finite number > 0"),
    (EXAMPLE, {"max_points": 1}, "max_points= must be >= 2"),
    (EXAMPLE, {"max_nodes": 0}, "max_nodes= must be >= 1"),
    (EXAMPLE, {"width": 0}, "width= must be >= 1"),
])
def test_refusals(model, kw, match):
    import jslpsolver_b200 as J
    with pytest.raises(ValueError, match=match):
        J.FrontierMIP(model, **kw)
    with pytest.raises(ValueError, match=match):
        FO.frontier_mip(model, **kw)


def test_frontier_still_refuses_mips():
    import jslpsolver_b200 as J
    with pytest.raises(ValueError, match="is defined for continuous LPs only"):
        J.Frontier(EXAMPLE)


# ---- C ABI --------------------------------------------------------------------------------------------------------
def test_box_batch_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    C, P = _lib.C, _lib.C.c_void_p
    want = ["jslp_tab *", "const jslp_scenario_edit *", "const int32_t *", "const jslp_cut *", "const int32_t *",
            "int", "int", "int", "int32_t *", "double *", "int32_t *", "int32_t *", "double *", "int32_t *",
            "double *", "int32_t *"]
    assert _types("jslp_box_batch") == want
    (_, res, got), = [s for s in _lib.SYMBOLS if s[0] == "jslp_box_batch"]
    assert res is C.c_int and got == [P] * 5 + [C.c_int] * 3 + [P] * 8

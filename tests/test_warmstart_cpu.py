"""CPU checks of the warm start (DESIGN.md section 2f): the oracle restatement (crash + simplex) against SciPy HiGHS on
every continuous fixture and on seeded mixed LPs after each kind of model edit, the round trip on an unchanged model,
the pivot saving on a perturbed dense packing LP, plan() on hand-built models, basis() as JSON, every refusal, and the
C prototype against the header."""
import copy
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT, load_bundle
from helpers import strip_timeouts

BUNDLE = load_bundle()


def _soft(jm):
    return any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())


CONTINUOUS = [f for f in BUNDLE["fixtures"] + BUNDLE["readme"]
              if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"]))
              and isinstance(f["model"].get("optimize"), str)]


def _host_model(jm):
    """The host Model of jm without a device tableau."""
    import jslpsolver_b200.tableau as T
    from jslpsolver_b200.model import Model
    saved = T.GpuTableau
    T.GpuTableau = lambda *a, **k: None
    try:
        return Model().loadJson(jm)
    finally:
        T.GpuTableau = saved


def _highs(jm):
    """linprog(HiGHS) of the JSON LP with unrestricted variables: ("optimal", result) / ("infeasible",) /
    ("unbounded",)."""
    from scipy.optimize import linprog
    names = list(jm["variables"])
    obj = jm["optimize"]
    kappa = -1.0 if jm.get("opType") == "max" else 1.0
    c = kappa * np.array([jm["variables"][v].get(obj, 0.0) for v in names], dtype=np.float64)
    A, b, Ae, be = [], [], [], []
    for cname, spec in jm["constraints"].items():
        a = np.array([jm["variables"][v].get(cname, 0.0) for v in names], dtype=np.float64)
        if spec.get("equal") is not None:
            Ae.append(a); be.append(spec["equal"])
            continue
        if spec.get("max") is not None:
            A.append(a); b.append(spec["max"])
        if spec.get("min") is not None:
            A.append(-a); b.append(-spec["min"])
    free = jm.get("unrestricted") or {}
    bounds = [(None, None) if free.get(v) else (0, None) for v in names]
    res = linprog(c, A_ub=np.array(A) if A else None, b_ub=np.array(b) if b else None,
                  A_eq=np.array(Ae) if Ae else None, b_eq=np.array(be) if be else None, bounds=bounds,
                  method="highs")
    if res.status == 0:
        return ("optimal", kappa * res.fun)
    if res.status == 2:
        return ("infeasible",)
    assert res.status == 3, res.message
    return ("unbounded",)


def _verdict(sol):
    if not sol.feasible:
        return ("infeasible",)
    if not sol.bounded:
        return ("unbounded",)
    return ("optimal", sol.evaluation)


def _agree(got, want, rel=1e-7):
    assert got[0] == want[0], (got, want)
    if got[0] == "optimal":
        assert abs(got[1] - want[1]) <= rel * max(1.0, abs(want[1])), (got, want)


def _cold_basis(jm):
    from oracle import ref_model, warmstart as W
    sol = ref_model.solve_full(jm, fast_cycles=True)
    assert sol.feasible and sol.bounded
    return W.basis(jm, sol), sol


# ---------------------------------------------------------------- seeded mixed LPs and their edits
def mixed_model(seed, n=12, m=10):
    """max or min over n non-negative variables (costs of both signs) with `min`, `max` and `equal` rows that a planted
    point satisfies, and `max` box rows that bound it.  (A warm start refuses unrestricted variables.)"""
    rng = np.random.default_rng(seed)
    names = [f"x{j}" for j in range(n)]
    free = {}
    x0 = {v: float(rng.uniform(0, 4)) for v in names}
    variables = {v: {"obj": float(rng.integers(-20, 21))} for v in names}
    constraints = {}
    for i in range(m):
        cname = f"row{i}"
        act = 0.0
        for v in names:
            if rng.random() < 0.6:
                a = float(rng.integers(-9, 10))
                variables[v][cname] = a
                act += a * x0[v]
        kind = rng.choice(["max", "min", "equal"], p=[0.5, 0.35, 0.15])
        if kind == "equal":
            constraints[cname] = {"equal": round(act, 6)}
        elif kind == "max":
            constraints[cname] = {"max": round(act + float(rng.uniform(0, 5)), 6)}
        else:
            constraints[cname] = {"min": round(act - float(rng.uniform(0, 5)), 6)}
    for v in names:
        variables[v]["box_" + v] = 1.0
        constraints["box_" + v] = {"min": 0.0, "max": 10.0} if v in free else {"max": 10.0}
    return {"optimize": "obj", "opType": "max" if seed % 2 else "min", "constraints": constraints,
            "variables": variables, "unrestricted": free}


def edit(jm, kind, seed):
    jm = copy.deepcopy(jm)
    rng = np.random.default_rng(seed + 1000)
    rows = [c for c in jm["constraints"] if not c.startswith("box_")]
    if kind == "coef":
        for v in jm["variables"].values():
            for k in v:
                if k != jm["optimize"] and not k.startswith("box_"):
                    v[k] = v[k] * (1 + 0.02 * float(rng.standard_normal()))
    elif kind == "rhs":
        for c in rows:
            spec = jm["constraints"][c]
            for side in spec:
                spec[side] = spec[side] + 0.5 * float(rng.standard_normal())
    elif kind == "cost":
        for v in jm["variables"].values():
            v[jm["optimize"]] = v[jm["optimize"]] * (1 + 0.1 * float(rng.standard_normal()))
    elif kind == "add_rows":
        for i in range(3):
            cname = f"new{i}"
            for v in jm["variables"].values():
                v[cname] = float(rng.integers(0, 5))
            jm["constraints"][cname] = {"max": float(rng.integers(20, 60))}
    elif kind == "add_vars":
        for j in range(3):
            v = f"y{j}"
            jm["variables"][v] = {jm["optimize"]: float(rng.integers(-10, 11)), "box_" + v: 1.0}
            jm["variables"][v].update({c: float(rng.integers(-5, 6)) for c in rows if rng.random() < 0.5})
            jm["constraints"]["box_" + v] = {"max": 5.0}
    elif kind == "del_rows":
        for c in rows[:3]:
            del jm["constraints"][c]
            for v in jm["variables"].values():
                v.pop(c, None)
    elif kind == "del_vars":
        for v in list(jm["variables"])[:3]:
            del jm["variables"][v]
            del jm["constraints"]["box_" + v]
            jm["unrestricted"].pop(v, None)
    elif kind == "rename":
        for c in rows[:2]:
            jm["constraints"]["renamed_" + c] = jm["constraints"].pop(c)
            for v in jm["variables"].values():
                if c in v:
                    v["renamed_" + c] = v.pop(c)
        for v in list(jm["variables"])[:2]:
            jm["variables"]["renamed_" + v] = jm["variables"].pop(v)
            if v in jm["unrestricted"]:
                jm["unrestricted"]["renamed_" + v] = jm["unrestricted"].pop(v)
    elif kind == "infeasible":
        for v in jm["variables"].values():
            v["wall"] = 1.0
        jm["constraints"]["wall"] = {"min": 1000.0}
    elif kind == "unbounded":
        sign = 1.0 if jm["opType"] == "max" else -1.0
        jm["variables"]["ray"] = {jm["optimize"]: sign * 3.0}
    else:
        raise KeyError(kind)
    return jm


def _reference_agrees(jm):
    """True when the reference's own cold solve reaches HiGHS's verdict on jm.  Its phase 1 has no artificial
    variables and can stop short of a feasible point on models with unrestricted variables; the warm start is held to
    HiGHS where the cold solve is."""
    from oracle import ref_model
    sol = ref_model.solve_full(jm, fast_cycles=True)
    h = _highs(jm)
    try:
        _agree(_verdict(sol), h)
        return True
    except AssertionError:
        return False


SEEDS = [s for s in range(60) if _reference_agrees(mixed_model(s))][:6]

EDITS = ["same", "coef", "rhs", "cost", "add_rows", "add_vars", "del_rows", "del_vars", "rename"]


def _warm_case(seed, kind):
    from oracle import warmstart as W
    jm = mixed_model(seed)
    b, _ = _cold_basis(jm)
    jm2 = jm if kind == "same" else edit(jm, kind, seed)
    sol, records, n, unknown = W.warm_solve(jm2, b)
    return jm2, b, sol, records, n, unknown


def test_fixtures_round_trip_against_highs():
    from oracle import ref_model, warmstart as W
    checked = 0
    for f in CONTINUOUS:
        jm = strip_timeouts(f["model"])
        cold = ref_model.solve_full(jm, fast_cycles=True)
        if not (cold.feasible and cold.bounded):
            continue
        b = W.basis(jm, cold)
        sol, records, n, unknown = W.warm_solve(jm, b)
        _agree(_verdict(sol), _highs(jm))
        assert unknown == {"variables": [], "constraints": []}
        checked += 1
    assert checked >= 10


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("kind", EDITS + ["infeasible", "unbounded"])
def test_mixed_edits_against_highs(seed, kind):
    jm2, b, sol, records, n, unknown = _warm_case(SEEDS[seed], kind)
    if kind in ("same", "infeasible", "unbounded") or _reference_agrees(jm2):
        _agree(_verdict(sol), _highs(jm2))
    if kind in ("rename", "del_rows", "del_vars"):  # names the edited model lacks are listed, never crashed
        assert set(unknown["variables"]) <= {v for v in b["variables"] if v not in jm2["variables"]}
        assert all(c["name"] not in jm2["constraints"] for c in unknown["constraints"])
    if kind in ("same", "coef", "rhs", "cost"):
        assert unknown == {"variables": [], "constraints": []}


@pytest.mark.parametrize("seed", range(6))
def test_round_trip_pivots_every_saved_variable(seed):
    from oracle import warmstart as W
    jm = mixed_model(SEEDS[seed])
    b, cold = _cold_basis(jm)
    sol, records, n, _ = W.warm_solve(jm, b)
    assert n == len(b["variables"])
    assert (records[:, 3] >= 0).all()
    assert abs(sol.evaluation - cold.evaluation) <= 1e-9 * max(1.0, abs(cold.evaluation))


def test_fixture_round_trip_pivots():
    from oracle import ref_model, warmstart as W
    for f in CONTINUOUS:
        jm = strip_timeouts(f["model"])
        cold = ref_model.solve_full(jm, fast_cycles=True)
        if not (cold.feasible and cold.bounded):
            continue
        b = W.basis(jm, cold)
        _, records, n, _ = W.warm_solve(jm, b)
        assert n == len(b["variables"]), f["name"] if "name" in f else jm


def test_dense_packing_noise_saves_pivots():
    """601 x 551 dense packing LP, every coefficient x (1 + 0.02 N(0,1)): crash + phase 1 + phase 2 pivots are at
    most a tenth of the cold solve's."""
    from jslpsolver_b200 import problems
    from oracle import ref_model, warmstart as W
    A, b, c = problems.dense_packing_lp_arrays(550, 600, 12345)
    jm = problems.lp_model(A, b, c)
    basis, cold = _cold_basis(jm)
    rng = np.random.default_rng(12346)
    jm2 = problems.lp_model(A * (1 + 0.02 * rng.standard_normal(A.shape)), b, c)
    cold2 = ref_model.solve_full(jm2, fast_cycles=True)
    sol, records, n, _ = W.warm_solve(jm2, basis)
    warm = n + sol.state.lastP1 + sol.state.lastP2
    assert warm * 10 <= cold2.state.lastP1 + cold2.state.lastP2
    assert abs(sol.evaluation - cold2.evaluation) <= 1e-7 * abs(cold2.evaluation)


# ---------------------------------------------------------------- plan() and basis()
HAND = {"optimize": "profit", "opType": "max",
        "constraints": {"a": {"max": 10}, "b": {"equal": 4}, "c": {"min": 1, "max": 8}},
        "variables": {"x": {"profit": 3, "a": 1, "b": 1, "c": 1}, "y": {"profit": 2, "a": 2, "c": 1},
                      "z": {"profit": 1, "b": 1}}}


def test_plan_order_mask_and_unknown_names():
    from jslpsolver_b200.warmstart import plan
    m = _host_model(HAND)
    idx = {c.name + ("+" if c.isUpperBound else "-"): c.index for c in m.constraints}
    vidx = {v.id: v.index for v in m.variables}
    b = {"variables": ["z", "nope", "x"],
         "constraints": [{"name": "b", "type": "max"}, {"name": "c", "type": "min"}, {"name": "gone", "type": "max"}]}
    enter, leave, unknown = plan(m, b)
    assert enter.tolist() == [vidx["z"], vidx["x"]]
    assert leave.dtype == np.uint8 and len(leave) == len(m.variables) + len(m.constraints)
    assert sorted(np.nonzero(leave)[0].tolist()) == sorted([idx["b+"], idx["c-"]])
    assert unknown == {"variables": ["nope"], "constraints": [{"name": "gone", "type": "max"}]}


def test_plan_programmatic_constraint_names():
    from jslpsolver_b200.warmstart import plan
    import jslpsolver_b200.tableau as T
    from jslpsolver_b200.model import Model
    saved = T.GpuTableau
    T.GpuTableau = lambda *a, **k: None
    try:
        m = Model()
        x = m.addVariable(1, "x")
        c0 = m.smallerThan(5).addTerm(1, x)
        c1 = m.greaterThan(1).addTerm(1, x)
    finally:
        T.GpuTableau = saved
    enter, leave, unknown = plan(m, {"variables": ["x"], "constraints": [{"name": c0.index, "type": "max"},
                                                                         {"name": c0.index, "type": "min"}]})
    assert enter.tolist() == [x.index]
    assert np.nonzero(leave)[0].tolist() == [c0.index]
    assert unknown["constraints"] == [{"name": c0.index, "type": "min"}]
    assert c1.index not in np.nonzero(leave)[0].tolist()


def test_basis_json_round_trip():
    from oracle import ref_model, warmstart as W
    from jslpsolver_b200.warmstart import plan
    sol = ref_model.solve_full(HAND, fast_cycles=True)
    b = W.basis(HAND, sol)
    assert json.loads(json.dumps(b)) == b
    assert set(b) == {"variables", "constraints"}
    assert all(set(c) == {"name", "type"} and c["type"] in ("max", "min") for c in b["constraints"])
    assert len(b["variables"]) == len(b["constraints"])  # a square basis: one binding row per basic structural
    _, _, unknown = plan(_host_model(HAND), b)
    assert unknown == {"variables": [], "constraints": []}
    warm, records, n, _ = W.warm_solve(HAND, b)
    assert n == len(b["variables"]) and warm.evaluation == sol.evaluation


@pytest.mark.parametrize("bad", [
    None, [], {"variables": []}, {"variables": [], "constraints": [], "x": 1}, {"variables": "x", "constraints": []},
    {"variables": [1.5], "constraints": []}, {"variables": [True], "constraints": []},
    {"variables": [], "constraints": [{"name": "a"}]}, {"variables": [], "constraints": [{"name": "a", "type": "eq"}]},
    {"variables": [], "constraints": ["a"]}, {"variables": [], "constraints": [{"name": None, "type": "max"}]}])
def test_malformed_basis_refused(bad):
    from jslpsolver_b200.warmstart import plan
    with pytest.raises(ValueError):
        plan(_host_model(HAND), bad)


def test_model_refusals():
    from jslpsolver_b200.warmstart import check_model
    ints = dict(HAND, ints={"x": 1})
    soft = dict(HAND, constraints=dict(HAND["constraints"], a={"max": 10, "weight": 2}))
    for jm in (ints, soft):
        with pytest.raises(ValueError):
            check_model(_host_model(jm))
    with pytest.raises(ValueError, match="unrestricted"):
        check_model(_host_model(dict(HAND, unrestricted={"x": 1})))
    m = _host_model(HAND)
    m.tableauInitialized = True
    with pytest.raises(ValueError, match="not been solved"):
        check_model(m)


def test_solve_refuses_before_any_device_work():
    """The refusals of Solve(basis=...) raise before a tableau is built, so they hold without a GPU."""
    from jslpsolver_b200.solver import Solve
    b = {"variables": [], "constraints": []}
    with pytest.raises(ValueError, match="multi-objective"):
        Solve(dict(HAND, optimize={"profit": "max", "a": "min"}), basis=b)
    with pytest.raises(ValueError):
        Solve(dict(HAND, ints={"x": 1}), basis=b)
    with pytest.raises(ValueError):
        Solve(HAND, basis={"variables": []})


def test_header_prototype_compiles():
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = ('#include "jslp_b200.h"\n'
           "int (*f)(jslp_tab *, const int32_t *, int, const uint8_t *, int32_t *, int *) = jslp_crash;\n")
    res = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                          "-x", "c", "-"], input=src, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr

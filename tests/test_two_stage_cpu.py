"""CPU checks of two-stage stochastic LPs (DESIGN.md section 2u): the restatement over the C oracle against SciPy HiGHS on
the deterministic equivalent (seeded capacity-expansion models with shared and per-case T, feasibility cuts, an
infeasible equivalent, an unbounded recourse, the farmer), the loop's properties, every refusal, the iteration limit and
the C prototype."""
import math
import os
import re

import pytest

from conftest import ROOT
import two_stage_models as TM
import two_stage_oracle as TO

SEEDED = [(seed, kw) for seed in range(4) for kw in ({}, {"per_case_t": True}, {"complete": False},
                                                     {"max_sense": True, "per_case_t": True})]


def _meets(model, names, values, rhs=None, tech=None, tol=1e-6):
    for n in names:
        spec = dict(model["constraints"][n])
        r = (rhs or {}).get(n)
        if isinstance(r, dict):
            spec.update(r)
        elif r is not None:
            spec = {k: r for k in spec if k in ("min", "max", "equal")}
        lhs = sum(float((tech or {}).get(n, {}).get(v, model["variables"][v].get(n, 0))) * x for v, x in values.items())
        scale = 1 + abs(lhs)
        if spec.get("max") is not None:
            assert lhs <= spec["max"] + tol * scale, (n, lhs, spec)
        if spec.get("min") is not None:
            assert lhs >= spec["min"] - tol * scale, (n, lhs, spec)
        if spec.get("equal") is not None:
            assert abs(lhs - spec["equal"]) <= tol * scale, (n, lhs, spec)


def _check_properties(model, cases, first, r):
    for it in r["iterations"]:
        assert it["lower"] <= it["upper"] + 1e-9 * (1 + abs(it["upper"])), it
    variables = model["variables"]
    second = [v for v in variables if v not in first]
    srows = [n for n in model["constraints"] if any(variables[y].get(n, 0) for y in second)]
    frows = [n for n in model["constraints"] if n not in srows]
    assert all(v >= -1e-9 for v in r["first"].values())
    _meets(model, frows, r["first"])
    for case, out in zip(cases, r["cases"]):
        assert set(out["values"]) == set(second)
        _meets(model, srows, dict(r["first"], **out["values"]), case.get("rhs"), case.get("coefficients"))


@pytest.mark.parametrize("seed,kw", SEEDED)
def test_seeded_models_match_highs(seed, kw):
    model, cases, first, p = TM.capacity(seed, **kw)
    status, want = TM.deterministic_equivalent(model, cases, first, p)
    r = TO.TwoStage(model, cases, first, p)
    assert status == 0 and r["stop"] == "reached" and r["exact"] and r["feasible"] and r["bounded"]
    assert r["result"] == pytest.approx(want, rel=1e-7, abs=1e-7)
    _check_properties(model, cases, first, r)
    total = sum(case["probability"] * case["result"] for case in r["cases"])
    assert total == pytest.approx(r["result"], rel=1e-9, abs=1e-9)
    if kw.get("complete") is False:
        assert sum(it["feasibility_cuts"] for it in r["iterations"]) > 0


def test_farmer():
    status, want = TM.deterministic_equivalent(TM.FARMER, TM.FARMER_CASES, TM.FARMER_FIRST)
    assert status == 0 and want == pytest.approx(108390, rel=1e-9)
    r = TO.TwoStage(TM.FARMER, TM.FARMER_CASES, TM.FARMER_FIRST)
    assert r["stop"] == "reached" and r["result"] == pytest.approx(108390, rel=1e-9)
    assert [round(r["first"][v], 6) for v in TM.FARMER_FIRST] == [170, 80, 250]
    _check_properties(TM.FARMER, TM.FARMER_CASES, TM.FARMER_FIRST, r)


def test_infeasible_equivalent():
    model, cases, first, p = TM.capacity(4, complete=False)
    assert TM.deterministic_equivalent(model, cases, first, p)[0] == 2
    r = TO.TwoStage(model, cases, first, p)
    assert r["stop"] == "infeasible" and not r["feasible"] and r["result"] is None and r["cases"] == []


def test_unbounded_recourse():
    model = {"optimize": "cost", "constraints": {"budget": {"max": 5}, "r": {"min": 1}},
             "variables": {"x": {"cost": 1, "budget": 1, "r": 1}, "y": {"cost": -1, "r": 1}}}
    cases = [{"rhs": {"r": 2}}, {"rhs": {"r": 3}}]
    assert TM.deterministic_equivalent(model, cases, ["x"])[0] == 3
    r = TO.TwoStage(model, cases, ["x"])
    assert r["stop"] == "unbounded" and not r["bounded"] and r["result"] == -math.inf
    # a case of probability 0 does not count
    model["variables"]["z"] = {"cost": 1, "r": 1}
    model["variables"]["y"] = {"cost": 1, "r": 1}
    assert TO.TwoStage(model, cases + [{"cost": {"y": -1}}], ["x"], [1, 1, 0])["stop"] == "reached"


def test_limit():
    model, cases, first, p = TM.capacity(1)
    r = TO.TwoStage(model, cases, first, p, max_iterations=1)
    assert r["stop"] == "limit" and not r["exact"] and len(r["iterations"]) == 1
    assert r["bound"] == -math.inf and r["result"] is not None


def test_refusals():
    model, cases, first, _ = TM.capacity(0)
    bad = [
        (dict(model, ints={"x0": 1}), cases, first, "integer"),
        (dict(model, binaries={"x0": 1}), cases, first, "binary"),
        (dict(model, unrestricted={"x0": 1}), cases, first, "unrestricted"),
        (dict(model, optimize={"cost": "min", "other": "max"}), cases, first, "one objective"),
        (dict(model, external={"solver": "x"}), cases, first, "external"),
        (dict(model, timeout=5), cases, first, "timeout"),
        (dict(model, options={"useMIRCuts": True}), cases, first, "useMIRCuts"),
        (dict(model, constraints=dict(model["constraints"], budget={"max": 9, "weight": 1})), cases, first, "soft"),
        (model, [], first, "non-empty"),
        (model, cases, ["nope"], "unknown variable"),
        (model, cases, list(model["variables"]), "every variable"),
        (model, [{"rhs": {"budget": 3}}], first, "first-stage row"),
        (model, [{"cost": {"x0": 3}}], first, "first-stage"),
        (model, [{"rhs": {"nope": 3}}], first, "nope"),
        (model, [{"cost": {"nope": 3}}], first, "nope"),
        (model, [{"other": 1}], first, "unknown case key"),
        (model, [{"coefficients": {"budget": {"x0": 1}}}], first, "first-stage row"),
        (model, [{"coefficients": {"nope": {"x0": 1}}}], first, "unknown constraint"),
        (model, [{"coefficients": {"link0": {"y0_0": 1}}}], first, "second-stage variable"),
        (model, [{"coefficients": {"link0": {"x0": float("nan")}}}], first, "finite"),
    ]
    for m, c, f, match in bad:
        with pytest.raises(ValueError, match=match):
            TO.TwoStage(m, c, f)
    for p in ([1], [1, -1, 1, 1, 1], [0, 0, 0, 0, 0], [1, 1, 1, 1, float("inf")]):
        with pytest.raises(ValueError, match="probabilit"):
            TO.TwoStage(model, cases, first, p)
    with pytest.raises(ValueError, match="max_iterations"):
        TO.TwoStage(model, cases, first, max_iterations=0)
    free = {"optimize": "cost", "constraints": {"r": {"min": 1}},
            "variables": {"x": {"cost": -1, "r": 1}, "y": {"cost": 1, "r": 1}}}
    with pytest.raises(ValueError, match="bound the first-stage variables"):
        TO.TwoStage(free, [{}], ["x"])


def test_internal_names_do_not_collide():
    model, cases, first, p = TM.capacity(2)
    model = dict(model, constraints=dict(model["constraints"], _two_stagecut0={"max": 1000}))
    model["variables"] = dict(model["variables"], x0=dict(model["variables"]["x0"], _two_stagecut0=1))
    status, want = TM.deterministic_equivalent(model, cases, first, p)
    assert TO.TwoStage(model, cases, first, p)["result"] == pytest.approx(want, rel=1e-7)


def test_ctypes_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+jslp_recourse_batch\s*\(([^)]*)\)\s*;", header)
    assert proto, "jslp_recourse_batch is not declared"
    params = [re.sub(r"\s+", " ", p.strip()) for p in proto.group(1).split(",")]
    types = [re.sub(r"\s*\b\w+$", "", p).replace(" *", "*") for p in params]
    want = ["jslp_tab*", "const jslp_scenario_edit*", "const int32_t*", "int", "const int32_t*", "int", "const double*",
            "int", "int", "int32_t*", "double*", "int32_t*", "int32_t*", "double*", "int32_t*", "double*", "double*"]
    assert types == want, types
    C = _lib.C
    (name, res, args), = [s for s in _lib.SYMBOLS if s[0] == "jslp_recourse_batch"]
    assert res is C.c_int and len(args) == len(want)
    for a, w in zip(args, want):
        assert (a is C.c_void_p) if w.endswith("*") else (a is C.c_int), (w, a)

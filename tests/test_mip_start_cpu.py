"""MIP starts (DESIGN.md section 2t) without a GPU: the restatement of tests/mip_start_oracle.py pinned to
orc_branch_and_cut when it has no starts; seeded runs against the cold run and SciPy's HiGHS `milp`; the host rules of
jslpsolver_b200/mipstart.py (zero convention, None, unknown names and head keys, continuous and presolve-fixed values,
fractional, skipped, incomplete, tie order); every refusal; and the jslp_branch_and_cut_start declaration and
jslp_start_status layout against their ctypes mirrors."""
from __future__ import annotations

import os
import subprocess

import numpy as np
import pytest

import mip_start_oracle as MSO
import pool_oracle as PO
from conftest import ROOT, load_bundle
from helpers import strip_timeouts
from jslpsolver_b200 import mipstart, problems
from jslpsolver_b200.model import Model
from jslpsolver_b200.model import presolve as product_presolve
from oracle.ref_model import RefModel, lib, presolve
from test_mip_variability_cpu import highs
from test_pool_cpu import _types


@pytest.fixture(scope="module", autouse=True)
def _oracle_lib():
    from oracle import ref_model
    ref_model.build_oracle()


def _plain_mip(jm: dict) -> bool:
    if not (jm.get("ints") or jm.get("binaries")) or not isinstance(jm.get("optimize"), str):
        return False
    return not any(isinstance(c, dict) and (c.get("weight") is not None or c.get("priority") is not None)
                   for c in jm["constraints"].values())


FIXTURES = [fx for fx in load_bundle()["fixtures"] if _plain_mip(fx["model"])]
FAMILIES = [problems.knapsack_mip_model(12, 4, seed=1), problems.knapsack_mip_model(16, 6, seed=2),
            problems.random_mip_model(14, 8, seed=3), problems.random_mip_model(18, 10, seed=5),
            problems.set_cover_model(12, 10, seed=4), problems.half_tie_mip_model(12, seed=6)]


def _ref(jm: dict) -> RefModel:
    model = RefModel().loadJson(jm)
    if model.usePresolve:
        infeasible, fixed = presolve(model)
        assert not infeasible
        for var in fixed:
            var.value, var.cost = fixed[var], 0
    return model


def _cold_oracle(model: RefModel):
    o = MSO.tableau(model)
    lib().orc_enable_node_log(o.h, 1 << 20)
    st = o.branch_and_cut()
    return o, st


def _feasible_presolve(jm: dict) -> bool:
    return not presolve(RefModel().loadJson(jm))[0]


@pytest.mark.parametrize("jm", [strip_timeouts(fx["model"]) for fx in FIXTURES] + FAMILIES,
                         ids=[fx["file"] for fx in FIXTURES] + [f"family{i}" for i in range(len(FAMILIES))])
def test_restatement_without_starts_is_the_oracle(jm):
    if not _feasible_presolve(jm):
        pytest.skip("presolve proves it infeasible: no branch and cut")
    o, st = _cold_oracle(_ref(jm))
    res = MSO.branch_and_cut(_ref(jm))
    assert np.array_equal(res["node_log"], o.node_log())
    fin = res["o"].state()
    assert (fin.evaluation, fin.feasible, fin.bounded) == (st.evaluation, st.feasible, st.bounded)
    assert res["iterations"] == st.bncIterations and res["is_integral"] == bool(st.isIntegral)
    assert res["best_cuts"] == o.best_cuts()
    assert np.array_equal(res["o"].matrix()[:, 0], o.matrix()[:, 0])
    assert np.array_equal(res["o"].maps()[0], o.maps()[0])


def _plan(simplified: dict, jm: dict) -> dict:
    return {k: v for k, v in simplified.items() if k in jm["variables"]}


def _pool_second(jm: dict):
    sols = PO.pool(jm, k=2)["solutions"]
    return None if len(sols) < 2 else {k: v for k, v in sols[1]["values"].items()}


def _tolerance(jm: dict):
    return jm.get("tolerance") or (jm.get("options") or {}).get("tolerance")


# the optimum is only defined with tolerance 0 (a tolerance stops the tree early)
SEEDED = FAMILIES + [strip_timeouts(fx["model"]) for fx in FIXTURES
                     if len(fx["model"]["variables"]) <= 40 and not _tolerance(fx["model"])]


@pytest.mark.parametrize("jm", SEEDED)
def test_seeded_runs_reach_the_cold_optimum(jm):
    if not _feasible_presolve(jm):
        pytest.skip("presolve proves it infeasible")
    cold, _, cres = MSO.solve(jm)
    m = Model().loadJson(jm)
    status, value = highs(jm, None, 0, None)
    if status == 0 and cold["feasible"]:
        assert cold["result"] == pytest.approx(value, rel=1e-9, abs=1e-9)
    plan = _plan(cold, jm)
    ints = [v.id for v in m.integerVariables]
    starts = {"optimal": plan, "result": dict(cold),
              "infeasible": {v: -1 for v in ints},  # x <= -1 on non-negative variables
              "partial": {**plan, **{v: None for v in ints[::2]}}}
    second = _pool_second(jm)
    if second is not None:
        starts["second"] = second
    for name, start in starts.items():
        seeded, report, res = MSO.solve(jm, start)
        assert seeded["feasible"] == cold["feasible"], name
        if cold["feasible"]:
            assert seeded["result"] == pytest.approx(cold["result"], rel=1e-9, abs=1e-9), name
        if name in ("optimal", "result") and report["seed"] is not None:
            assert res["iterations"] <= cres["iterations"], name  # DESIGN.md section 2t on the bound
            assert not report["improved"]
        if name == "infeasible" and report["starts"][0]["status"] != "skipped" and not m.unrestrictedVariables:
            assert report["starts"][0]["status"] == "infeasible" and report["seed"] is None


KNAP = {"optimize": "v", "opType": "max", "constraints": {"w": {"max": 10}},
        "variables": {"a": {"w": 5, "v": 6}, "b": {"w": 4, "v": 5}, "c": {"w": 3, "v": 3}, "x": {"w": 1, "v": 0.5}},
        "ints": {"a": 1, "b": 1, "c": 1}}


def _mapped(jm, start):
    m = Model().loadJson(jm)
    m.presolveResult = product_presolve(m)
    return m, mipstart.cut_lists(m, mipstart.plans(start))


def test_zero_convention_none_unknown_and_head_keys():
    m, (s,) = _mapped(KNAP, {"a": 1, "c": None, "zz": 3, "feasible": True, "result": 9, "bounded": True,
                             "isIntegral": True})
    ia, ib = (v.index for v in m.integerVariables[:2])
    assert s["cuts"] == [(0, ia, 1.0), (1, ia, 1.0), (1, ib, 0.0)]  # b missing = 0; c free
    assert s["unknown"] == ["zz"] and s["ignored"] == []
    jm = {**KNAP, "variables": {**KNAP["variables"], "result": {"w": 1, "v": 1}}, "ints": {**KNAP["ints"], "result": 1}}
    m, (s,) = _mapped(jm, {"result": 2})
    assert (0, m.integerVariables[-1].index, 2.0) in s["cuts"]


def test_continuous_and_presolve_fixed_values_are_ignored():
    jm = {**KNAP, "constraints": {**KNAP["constraints"], "fixc": {"max": 0}},
          "variables": {**KNAP["variables"], "c": {"w": 3, "v": 3, "fixc": 1}}}
    m, (s,) = _mapped(jm, {"x": 1.5, "c": 1, "a": 1})
    assert s["ignored"] == ["x", "c"]
    assert all(cut[1] != m.variables[2].index for cut in s["cuts"])


def test_fractional_start_is_rejected_on_the_host():
    _, (s, t) = _mapped(KNAP, [{"a": 0.5}, {"a": 1 + 1e-12}])
    assert s["cuts"] is None and t["cuts"] is not None
    _, report, _ = MSO.solve(KNAP, [{"a": 0.5}])
    assert report["starts"][0]["status"] == "fractional" and report["seed"] is None


def test_skipped_when_the_root_is_integral_or_infeasible():
    integral = {"optimize": "v", "opType": "max", "constraints": {"w": {"max": 4}},
                "variables": {"a": {"w": 1, "v": 1}}, "ints": {"a": 1}}
    _, report, _ = MSO.solve(integral, {"a": 4})
    assert report["starts"][0]["status"] == "skipped"
    infeasible = {"optimize": "v", "opType": "max", "constraints": {"w": {"max": 4}, "d": {"min": 5}},
                  "variables": {"a": {"w": 1, "d": 1, "v": 1}, "b": {"w": 1, "d": 1, "v": 1}},
                  "ints": {"a": 1, "b": 1}, "options": {"presolve": False}}
    res, report, _ = MSO.solve(infeasible, {"a": 1})
    assert not res["feasible"] and report["starts"][0]["status"] == "skipped"


def test_incomplete_at_start_nodes_one():
    _, report, _ = MSO.solve(KNAP, {"a": None, "b": None, "c": None}, start_nodes=1)
    assert report["starts"][0]["status"] == "incomplete" and report["starts"][0]["nodes"] == 1


def test_seed_wins_ties_and_the_lowest_index_wins_among_starts():
    tie = {"optimize": "v", "opType": "max", "constraints": {"w": {"max": 3}},
           "variables": {"a": {"w": 2, "v": 2}, "b": {"w": 2, "v": 2}, "c": {"w": 2.5, "v": 1}},
           "ints": {"a": 1, "b": 1, "c": 1}}
    cold, _, _ = MSO.solve(tie)
    for plan in ({"b": 1}, {"a": 1}):
        res, report, _ = MSO.solve(tie, [{"c": 1}, plan, {"a": 1} if plan == {"b": 1} else {"b": 1}])
        assert res["result"] == cold["result"] == 2
        assert report["seed"] == 1 and not report["improved"]
        assert [s["status"] for s in report["starts"]] == ["feasible", "seed", "feasible"]
        assert {k: v for k, v in res.items() if k in "ab"} == plan  # the seed's completion is returned


@pytest.mark.parametrize("model, kw, match", [
    ({"optimize": "v", "constraints": {"w": {"max": 1}}, "variables": {"x": {"w": 1, "v": 1}}}, {}, "continuous"),
    (KNAP, {"basis": {"variables": [], "constraints": []}}, "basis"),
    ({**KNAP, "constraints": {"w": {"max": 10, "weight": 2}}}, {}, "soft constraints"),
    ({**KNAP, "constraints": {"w": {"max": 10, "priority": "strong"}}}, {}, "soft constraints"),
    ({**KNAP, "optimize": {"v": "max", "w": "min"}}, {}, "multi-objective"),
    ({**KNAP, "external": {"solver": "x"}}, {}, "external"),
    ({**KNAP, "options": {"nodeSelection": "best-first"}}, {}, "default branch-and-cut service"),
    ({**KNAP, "options": {"branching": "strong"}}, {}, "default branch-and-cut service"),
    ({**KNAP, "options": {"useIncremental": True}}, {}, "default branch-and-cut service"),
    (KNAP, {"start_nodes": 0}, "start_nodes"),
    (KNAP, {"start": 3}, "dict"),
])
def test_refusals(model, kw, match):
    import jslpsolver_b200 as J
    kw = {"start": {"a": 1}, **kw}
    with pytest.raises(ValueError, match=match):
        J.Solve(model, **kw)


def test_distributed_is_refused():
    m = Model().loadJson(KNAP)
    m.tableau.distributed = True
    with pytest.raises(ValueError, match="one GPU"):
        m.solve(start={"a": 1})


def test_start_signature_and_struct_match_the_header(tmp_path):
    import ctypes as C
    from jslpsolver_b200 import _lib
    P = C.c_void_p
    assert _types("jslp_branch_and_cut_start") == [
        "jslp_tab *", "const jslp_bnb_opts *", "const jslp_cut *", "const int32_t *", "int", "int64_t",
        "jslp_start_status *", "jslp_bnb_status *", "jslp_cut *", "int"]
    (_, res, got), = [s for s in _lib.SYMBOLS if s[0] == "jslp_branch_and_cut_start"]
    assert res is C.c_int and got == [P, C.POINTER(_lib.BnbOpts), P, P, C.c_int, C.c_int64, P,
                                      C.POINTER(_lib.BnbStatus), P, C.c_int]
    cls = _lib.StartStatus
    src = tmp_path / "start.c"
    src.write_text("\n".join(
        ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "jslp_b200.h")}"',
         "int main(void) {", 'printf("%zu\\n", sizeof(jslp_start_status));'] +
        [f'printf("%zu\\n", offsetof(jslp_start_status, {f}));' for f, _ in cls._fields_] +
        [f'printf("%d\\n", {e});' for e in ("JSLP_START_SEED", "JSLP_START_FEASIBLE", "JSLP_START_INFEASIBLE",
                                              "JSLP_START_INCOMPLETE", "JSLP_START_SKIPPED")] + ["return 0; }"]))
    exe = tmp_path / "start"
    subprocess.run(["gcc", "-std=c11", "-o", str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got[:1 + len(cls._fields_)] == [C.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_]
    assert got[1 + len(cls._fields_):] == [_lib.START_SEED, _lib.START_FEASIBLE, _lib.START_INFEASIBLE,
                                           _lib.START_INCOMPLETE, _lib.START_SKIPPED]
    assert mipstart.STATUS[_lib.START_SEED] == "seed" and mipstart.STATUS[_lib.START_SKIPPED] == "skipped"

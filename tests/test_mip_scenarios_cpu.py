"""What-if scenarios of a MIP (DESIGN.md section 2p) without a GPU: the oracle restatement (tests/mip_scenarios_oracle.py)
against SciPy's HiGHS on the bundle's small MIPs and on generated MIPs, infeasible and unbounded cases included; the
product's commit rule (jslp_bnb::Tree, built with g++) fed the oracle's node results against the oracle's own branch and
cut, node log for node log; the edited models, their column 0 and row 0 against the edited initial tableau bit for bit;
the refusals; and the C ABI declaration."""
from __future__ import annotations

import math
import os
import random
import subprocess

import numpy as np
import pytest

import mip_scenarios_oracle as SO
from helpers import highs_solve, strip_timeouts
from jslpsolver_b200 import mip_scenarios as MS, problems
from jslpsolver_b200.model import Model
from test_pool_cpu import _types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def seeded_cases(jm: dict, n: int, seed: int, spread: float = 0.2) -> list:
    """n cases of seeded right-hand-side and cost perturbations of jm: every constraint with a finite bound moves by up
    to `spread` of its value (a min+max constraint as {"min", "max"}), and up to three objective coefficients move."""
    rng = random.Random(seed)
    cons = [(name, spec) for name, spec in jm["constraints"].items() if isinstance(spec, dict)]
    objective = jm.get("optimize")
    priced = [vid for vid, coefs in jm["variables"].items() if isinstance(coefs.get(objective), (int, float))]
    out = []
    for _ in range(n):
        rhs = {}
        for name, spec in rng.sample(cons, min(len(cons), 3)):
            move = lambda v: float(round(v * (1 + rng.uniform(-spread, spread)), 3))  # noqa: E731
            if spec.get("equal") is not None:
                rhs[name] = move(spec["equal"])
            elif spec.get("min") is not None and spec.get("max") is not None:
                lo = move(spec["min"])
                rhs[name] = {"min": lo, "max": max(lo, move(spec["max"]))}
            elif spec.get("min") is not None:
                rhs[name] = move(spec["min"])
            elif spec.get("max") is not None:
                rhs[name] = move(spec["max"])
        cost = {vid: float(round(jm["variables"][vid][objective] * (1 + rng.uniform(-spread, spread)), 3))
                for vid in rng.sample(priced, min(len(priced), 3))}
        out.append({"rhs": rhs, "cost": cost})
    return out


def base_and_edited(jm: dict, spec: dict):
    m = Model().loadJson(dict(jm, options={"presolve": False}))
    return m, MS.edited(jm, m, spec)


EQUAL = {"optimize": "v", "opType": "max", "constraints": {"e": {"equal": 7}, "c": {"max": 10}},
         "variables": {"a": {"v": 3, "e": 1, "c": 2}, "b": {"v": 2, "e": 1, "c": 1}}, "ints": {"a": 1}}
RANGE = {"optimize": "cost", "opType": "min", "constraints": {"r": {"min": 2, "max": 9}, "s": {"min": 1}},
         "variables": {"a": {"cost": 4, "r": 1, "s": 1}, "b": {"cost": 3, "r": 2}}, "ints": {"a": 1, "b": 1}}
MAXED = {"optimize": "profit", "opType": "max",
         "constraints": {"wood": {"max": 300}, "labor": {"max": 110}},
         "variables": {"table": {"wood": 30, "labor": 5, "profit": 1200},
                       "dresser": {"wood": 20, "labor": 10, "profit": 1600}},
         "binaries": {"table": 1}, "ints": {"dresser": 1}}


@pytest.mark.parametrize("jm, spec", [
    (EQUAL, {"rhs": {"e": 5.5}, "cost": {"b": 0.1}}),
    (RANGE, {"rhs": {"r": {"min": 3, "max": 3.25}, "s": 0.1}, "cost": {"a": -1}}),
    (RANGE, {"rhs": {"r": {"max": 100}}}),
    (MAXED, {"rhs": {"wood": 299.9}, "cost": {"table": 1200.5, "dresser": 0}}),
])
def test_edges_are_the_edited_tableau_bit_for_bit(jm, spec):
    m, ed = base_and_edited(jm, spec)
    base, it = m.initial_tableau(), Model().loadJson(ed).initial_tableau()
    c0, r0 = MS.edges(base, it)
    assert np.array_equal(c0.view(np.uint64), it.matrix[:, 0].view(np.uint64))
    assert np.array_equal(r0.view(np.uint64), it.matrix[0].view(np.uint64))
    # the base with the edges written over it is the edited tableau, every bit of it
    rebuilt = base.matrix.copy()
    rebuilt[1:, 0] = c0[1:]
    rebuilt[0, :] = r0
    assert np.array_equal(rebuilt.view(np.uint64), it.matrix.view(np.uint64))
    assert ed["options"]["presolve"] is False and "presolve" not in (jm.get("options") or {})


def test_edited_writes_values_not_differences():
    jm = {"optimize": "v", "opType": "min", "constraints": {"c": {"min": 0.1}},
          "variables": {"a": {"v": 1, "c": 1}}, "ints": {"a": 1}}
    _, ed = base_and_edited(jm, {"rhs": {"c": 0.7}})
    assert ed["constraints"]["c"]["min"] == 0.7 and jm["constraints"]["c"]["min"] == 0.1


def test_edges_refuse_any_other_difference():
    m, ed = base_and_edited(RANGE, {"rhs": {"s": 2}})
    base = m.initial_tableau()
    it = Model().loadJson(ed).initial_tableau()
    it.matrix[1, 1] = np.nextafter(it.matrix[1, 1], np.inf)
    with pytest.raises(ValueError, match="changes more than"):
        MS.edges(base, it)
    it = Model().loadJson(ed).initial_tableau()
    it.integerIndices = it.integerIndices[:1]
    with pytest.raises(ValueError, match="changes more than"):
        MS.edges(base, it)


@pytest.mark.parametrize("model, cases, match", [
    (dict(MAXED, optimize={"profit": "max", "wood": "min"}), [], "one objective"),
    (dict(MAXED, constraints={"wood": {"max": 300, "weight": 2}}), [], "soft constraints"),
    (dict(MAXED, external={"solver": "lpsolve"}), [], "external"),
    (dict(MAXED, options={"useMIRCuts": True}), [], "useMIRCuts"),
    (dict(MAXED, options={"nodeSelection": "best-first"}), [], "nodeSelection"),
    (dict(MAXED, options={"branching": "pseudocost"}), [], "branching"),
    (dict(MAXED, options={"useIncremental": True}), [], "useIncremental"),
    (dict(MAXED, options={"keep_solutions": True}), [], "keep_solutions"),
    (dict(MAXED, options={"timeout": 100}), [], "timeout"),
    (dict(MAXED, timeout=100), [], "timeout"),
    (MAXED, {"rhs": {}}, "list of scenarios"),
    (MAXED, [{"bounds": {}}], "unknown scenario key"),
    (MAXED, [{"rhs": {"nails": 3}}], "no constraint named 'nails'"),
    (MAXED, [{"cost": {"chair": 3}}], "no variable named 'chair'"),
    (MAXED, [{"rhs": {"wood": float("nan")}}], "finite number"),
    (MAXED, [{"rhs": {"wood": {"min": 3}}}], "only a 'max' bound"),
    (MAXED, [{"rhs": {"wood": {}}}], "needs a 'min' and / or a 'max'"),
    (RANGE, [{"rhs": {"r": 4}}], "has a min and a max bound"),
    (EQUAL, [{"rhs": {"e": {"min": 3}}}], "is an equality: give one value"),
    (MAXED, [{"rhs": {"wood": 3}}, {"cost": {"table": True}}], "finite number"),
])
def test_refusals(model, cases, match):
    import jslpsolver_b200 as J
    with pytest.raises(ValueError, match=match):
        J.Scenarios(model, cases)


def test_no_cases_and_the_caller_model_unchanged():
    import copy
    import jslpsolver_b200 as J
    jm = copy.deepcopy(RANGE)
    assert J.Scenarios(jm, []) == []
    for spec in seeded_cases(jm, 4, seed=3):
        MS.edited(jm, Model().loadJson(jm), spec)
    assert jm == RANGE


def test_seeded_cases_are_valid_on_every_small_mip_fixture():
    from conftest import load_bundle
    b = load_bundle()
    for f in b["fixtures"] + b["readme"]:
        jm = f["model"]
        if not (jm.get("ints") or jm.get("binaries")) or len(jm["variables"]) > 200:
            continue
        m = Model().loadJson(dict(jm, options=dict(jm.get("options") or {}, presolve=False)))
        base = m.initial_tableau()
        for spec in seeded_cases(jm, 3, seed=11):
            MS.edges(base, Model().loadJson(MS.edited(jm, m, spec)).initial_tableau())


def test_bnb_batch_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    C, P = _lib.C, _lib.C.c_void_p
    want = ["jslp_tab *", "const double *", "const double *", "int", "const jslp_bnb_opts *", "int",
            "jslp_bnb_status *", "double *", "int32_t *", "int32_t *"]
    assert _types("jslp_bnb_batch") == want
    (_, res, got), = [s for s in _lib.SYMBOLS if s[0] == "jslp_bnb_batch"]
    assert res is C.c_int and got == [P, P, P, C.c_int, C.POINTER(_lib.BnbOpts), C.c_int, P, P, P, P]


def test_edited_reads_a_one_key_optimize_dict():
    jm = dict(MAXED, optimize={"profit": "max"})
    jm.pop("opType")
    _, ed = base_and_edited(MS._one_objective(jm), {"cost": {"table": 1000}})
    ed2 = MS.edited(jm, Model().loadJson(MS._one_objective(jm)), {"cost": {"table": 1000}})
    assert ed2 == ed and ed2["optimize"] == "profit" and ed2["opType"] == "max"
    assert ed2["variables"]["table"]["profit"] == 1000


# ---- the oracle restatement against HiGHS ----------------------------------------------------------------------------
def assert_matches_highs(jm: dict, cases: list):
    got = SO.scenarios(jm, cases)
    base = SO.base_model(jm)
    for spec, r in zip(cases, got):
        ed = MS.edited(jm, base, spec)
        status, obj = highs_solve(ed)
        if status == 0:
            assert r["feasible"] and r["bounded"], (spec, r)
            assert math.isclose(r["result"], obj, rel_tol=1e-6, abs_tol=1e-6), (spec, r["result"], obj)
        elif status == 2:
            assert not r["feasible"], (spec, r)
        else:  # unbounded (or unbounded-or-infeasible): the root relaxation is unbounded
            assert not r["bounded"] or not r["feasible"], (spec, r)


def test_restatement_matches_highs_on_small_mip_fixtures():
    from conftest import load_bundle
    b = load_bundle()
    n = 0
    for i, f in enumerate(b["fixtures"] + b["readme"]):
        jm = f["model"]
        # a relative tolerance stops branch and cut short of the optimum by design
        if not (jm.get("ints") or jm.get("binaries")) or not jm.get("optimize") or len(jm["variables"]) > 64 or \
                jm.get("tolerance") or \
                (jm.get("options") or {}).get("tolerance"):
            continue
        jm = strip_timeouts(jm)
        assert_matches_highs(jm, seeded_cases(jm, 3, seed=300 + i))
        n += 1
    assert n >= 8


@pytest.mark.parametrize("jm", [problems.random_mip_model(8, 6, seed=s) for s in (1, 2, 3)] +
                         [problems.knapsack_mip_model(10, 3, seed=s) for s in (4, 5)] +
                         [problems.set_cover_model(10, 8, seed=6)], ids=lambda m: m.get("name", "gen"))
def test_restatement_matches_highs_on_generated_mips(jm):
    assert_matches_highs(jm, seeded_cases(jm, 6, seed=7, spread=0.3))


def test_restatement_matches_highs_on_infeasible_and_unbounded_cases():
    parity = {"optimize": "v", "opType": "max", "constraints": {"odd": {"equal": 3}, "cap": {"max": 10}},
              "variables": {"a": {"v": 1, "odd": 2, "cap": 1}, "b": {"v": 1, "odd": 2, "cap": 1}},
              "ints": {"a": 1, "b": 1}}
    assert_matches_highs(parity, [{"rhs": {"odd": 4}}, {"rhs": {"odd": 5}}, {"rhs": {"cap": 1}}, {}])
    open_top = {"optimize": "v", "opType": "max", "constraints": {"c": {"min": 1}, "d": {"max": 5}},
                "variables": {"a": {"v": 1, "c": 1}, "b": {"v": 1, "c": 1, "d": 1}}, "ints": {"a": 1}}
    assert_matches_highs(open_top, [{"cost": {"a": -1}}, {}, {"rhs": {"d": 0}, "cost": {"a": -1, "b": 2}}])


# ---- the shared commit rule against the oracle's branch and cut --------------------------------------------------------
def replay_tree(exe, jm: dict, width: int = 1):
    """(node log, iterations, best cut count) of jslp_bnb::Tree over jm (presolve off), speculating `width` nodes a round
    after the root, every node evaluated by the oracle from the root snapshot (restore it, append the cuts, simplex)."""
    from oracle import ref_model as R
    model = R.RefModel().loadJson(jm)
    M, vrow, vcol, _, rc = model.build_tableau()
    tab = R.OracleTableau(M, vrow, vcol, precision=model.precision, integers=[v.index for v in model.integerVariables],
                          check_cycles=model.checkForCycles, is_min=model.isMinimization)
    p = subprocess.Popen([str(exe)], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
    p.stdin.write(f"{float(model.tolerance or 0)!r} {int(model.isMinimization)} 0 {width}\n")
    p.stdin.flush()
    while True:
        line = p.stdout.readline().split()
        if line[0] == "EVAL":
            v = line[2:]
            cuts = [(int(v[3 * i]), int(v[3 * i + 1]), float(v[3 * i + 2])) for i in range(int(line[1]))]
            before = tab.state().totalPivots
            st = tab.apply_cuts(cuts)
            integral = int(st.feasible and tab.is_integral())
            var, val = tab.most_fractional() if st.feasible and not integral else (-1, 0.0)
            optimal = int(st.feasible and st.bounded)
            p.stdin.write(f"{st.feasible} {st.bounded} {optimal} {integral} {var} {val!r} {st.evaluation!r} "
                          f"{st.totalPivots - before}\n")
            p.stdin.flush()
        elif line[0] == "SAVE":
            tab.save()
            p.stdin.write("ok\n")
            p.stdin.flush()
        elif line[0] == "LOG":
            log = np.array([[float(x) for x in p.stdout.readline().split()] for _ in range(int(line[1]))])
            it, nbest = (int(x) for x in p.stdout.readline().split()[1:])
            p.wait()
            return log.reshape(-1, 8), it, nbest


@pytest.fixture(scope="module")
def tree_exe(tmp_path_factory):
    exe = tmp_path_factory.mktemp("tree") / "tree_replay"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(ROOT, "jslpsolver_b200", "csrc"), "-o", str(exe),
                    os.path.join(ROOT, "tests", "cpp", "tree_replay.cpp")], check=True)
    return exe


def test_commit_rule_reproduces_the_oracle_node_log(tree_exe):
    """At every speculation width the commits, and so the node log, are the oracle's bit for bit."""
    from conftest import load_bundle
    from oracle import ref_model as R
    b = load_bundle()
    models = [strip_timeouts(f["model"]) for f in b["fixtures"] + b["readme"]
              if (f["model"].get("ints") or f["model"].get("binaries")) and len(f["model"]["variables"]) <= 64]
    models += [problems.random_mip_model(8, 6, seed=s) for s in (1, 2, 3)]
    models += [problems.knapsack_mip_model(10, 3, seed=4)]
    for jm in models:
        for spec in [{}] + seeded_cases(jm, 2, seed=9):
            ed = MS.edited(jm, SO.base_model(jm), spec)
            sol = R.solve_full(ed, node_log=1 << 16)
            want = sol.tableau.node_log()
            for width in (1, 2, 16):
                log, it, nbest = replay_tree(tree_exe, ed, width)
                assert it == sol.iter, (jm.get("name"), spec, width)
                assert log.shape == want.shape and np.array_equal(log.view(np.uint64), want.view(np.uint64)), \
                    (jm.get("name"), spec, width)
                assert nbest == len(sol.tableau.best_cuts()) or not sol.state.isIntegral

"""What-if scenarios of a MIP on the H100 (DESIGN.md section 2p): Scenarios() equals [Solve(edited_k) ...] dict for dict
on every MIP fixture of the bundle with seeded cases, at every width and on both node paths; per scenario, the counters,
evaluation bits and final column 0 of jslp_bnb_batch equal a separate jslp_branch_and_cut run on the edited tableau;
and the edge cases: infeasible and unbounded roots, a root integral at once, a cycling scenario, a continuous LP, more
trees than one launch holds, a log cap that forces redo, and the caller's tab left as it was."""
from __future__ import annotations

import numpy as np
import pytest

from jslpsolver_b200 import _lib, mip_scenarios as MS, problems
from jslpsolver_b200.model import Model
import mip_scenarios_oracle as SO
from helpers import strip_timeouts
from test_gpu_pool import beale_mip, mip_fixtures
from test_mip_scenarios_cpu import seeded_cases

pytestmark = pytest.mark.gpu


def solver(engine: int = 0, options=None):
    import jslpsolver_b200 as J
    s = J.Solver()
    s.engine = engine
    s.options.update(options or {})
    return s


def assert_equals_solve(jm: dict, cases: list, s=None, **kw):
    s = s or solver()
    got = s.Scenarios(jm, cases, **kw)
    base = Model().loadJson(dict(jm, options={"presolve": False}))
    want = [s.Solve(MS.edited(jm, base, spec)) for spec in cases]
    assert len(got) == len(want)
    for k, (g, w) in enumerate(zip(got, want)):
        assert g == w and list(g) == list(w), (jm.get("name"), k, cases[k], g, w)
    return got


def small(jm: dict) -> bool:
    return len(jm["variables"]) <= 200


def test_every_mip_fixture_equals_solve():
    for i, jm in enumerate(mip_fixtures()):
        if small(jm):  # a wall-clock stop is refused (DESIGN.md 2p)
            jm = strip_timeouts(jm)
            cases = seeded_cases(jm, 2, seed=100 + i)
            got = assert_equals_solve(jm, cases)
            if len(jm["variables"]) <= 64:  # the restatement over the C oracle (tests/mip_scenarios_oracle.py)
                assert got == SO.scenarios(jm, cases), jm.get("name")


def test_single_tableau_engine_equals_solve():
    """Engine 2: every root and node on the single-tableau path."""
    for i, jm in enumerate(mip_fixtures()):
        if len(jm["variables"]) <= 31:
            assert_equals_solve(strip_timeouts(jm), seeded_cases(jm, 3, seed=200 + i), solver(2))


@pytest.mark.parametrize("width", [1, 4, 16, 64])
def test_widths_give_identical_results(width):
    jm = problems.knapsack_mip_model(12, 3, seed=7)
    cases = seeded_cases(jm, 24, seed=5)
    assert_equals_solve(jm, cases, width=width)


def status_against_branch_and_cut(jm: dict, cases: list, s=None):
    """jslp_bnb_batch per scenario against jslp_branch_and_cut on the edited model's own tableau; the caller's tableau,
    both label arrays included, is left as it was."""
    base_m = Model().loadJson(dict(jm, options={"presolve": False}))
    base = base_m.initial_tableau()
    edges = [MS.edges(base, Model().loadJson(MS.edited(jm, base_m, spec)).initial_tableau()) for spec in cases]
    s = s or solver()
    inst = s._instance(dict(jm, options={"presolve": False}), None)
    tab = inst.tableau
    tab.setModel(inst)
    before, vrow, vcol = tab.matrix2d().copy(), tab.varIndexByRow.copy(), tab.varIndexByCol.copy()
    out = tab.bnb_batch(np.array([c for c, _ in edges]), np.array([r for _, r in edges]),
                        tolerance=float(inst.tolerance or 0))
    tab._refresh_dims()
    assert (tab.height, tab.width) == before.shape
    assert np.array_equal(tab.matrix2d().view(np.uint64), before.view(np.uint64))  # the caller's tab as it was
    assert np.array_equal(tab.varIndexByRow, vrow) and np.array_equal(tab.varIndexByCol, vcol)
    for k, spec in enumerate(cases):
        one = s._instance(MS.edited(jm, base_m, spec), None)
        one.tableau.setModel(one)
        one.tableau.branchAndCut()
        st, got = one.tableau.lastBnbStatus, out["status"][k]
        for f in ("feasible", "bounded", "is_integral", "iterations", "n_best_cuts"):
            assert getattr(got, f) == getattr(st, f), (k, f, getattr(got, f), getattr(st, f))
        assert np.float64(got.evaluation).tobytes() == np.float64(st.evaluation).tobytes(), k
        assert np.float64(got.best_possible_eval).tobytes() == np.float64(st.best_possible_eval).tobytes(), k
        if st.iterations > 0:
            assert got.pivots == st.pivots, k
        h = int(out["height"][k])
        assert h == one.tableau.height, k
        assert np.array_equal(out["rhs"][k, :h].view(np.uint64), one.tableau.rhs_column().view(np.uint64)), k
        assert np.array_equal(out["vrow"][k, :h], one.tableau.varIndexByRow), k
        one.tableau.close()
    tab.close()


def test_counters_and_final_column_equal_branch_and_cut():
    for seed in (1, 2):
        jm = problems.random_mip_model(10, 6, seed=seed)
        status_against_branch_and_cut(jm, seeded_cases(jm, 6, seed=seed))
    jm = problems.set_cover_model(12, 10, seed=3)
    status_against_branch_and_cut(jm, seeded_cases(jm, 6, seed=3))


@pytest.mark.parametrize("s", [solver(2), solver(options={_lib.OPT_NODE_LOG_CAP: 2})], ids=["engine2", "logcap2"])
def test_single_tableau_path_leaves_the_caller_tab(s):
    """Every root and node on the single-tableau path (engine 2), or redone there (a log cap of 2)."""
    for seed in (1, 2):
        jm = problems.random_mip_model(10, 6, seed=seed)
        status_against_branch_and_cut(jm, seeded_cases(jm, 4, seed=seed), s)


def test_log_cap_forces_redo_on_the_single_tableau_path():
    jm = problems.knapsack_mip_model(12, 3, seed=9)
    assert_equals_solve(jm, seeded_cases(jm, 8, seed=2), solver(options={_lib.OPT_NODE_LOG_CAP: 2}))


def test_more_trees_than_one_launch_holds():
    """4100 roots: more CTAs than batch_chunk allows in one launch (4096), so the roots span two launches."""
    jm = {"optimize": "profit", "opType": "max", "constraints": {"wood": {"max": 300}, "labor": {"max": 110}},
          "variables": {"table": {"wood": 30, "labor": 5, "profit": 1200},
                        "dresser": {"wood": 20, "labor": 10, "profit": 1600}}, "ints": {"table": 1, "dresser": 1}}
    cases = seeded_cases(jm, 4100, seed=8)
    s = solver()
    got = s.Scenarios(jm, cases)
    base = Model().loadJson(dict(jm, options={"presolve": False}))
    for k in list(range(0, 4100, 97)) + [4095, 4096, 4099]:
        assert got[k] == s.Solve(MS.edited(jm, base, cases[k])), k


def max_resident_height(W: int) -> int:
    """The tallest node the shared-memory node kernel takes at width W (node_smem_bytes / resident_fits)."""
    import torch
    optin = getattr(torch.cuda.get_device_properties(0), "shared_memory_per_block_optin", 232448)
    Ws = (W + 1) & ~1
    h = 1
    while 8 * ((h + 1) * Ws + 2 * Ws + (h + 1) + 1) + 16 * (h + 1) + 4 * (2 * (h + 1) + W) + 16 <= optin - 4096:
        h += 1
    return h


def test_resident_and_too_tall_nodes_in_one_round():
    """A knapsack base one row below the shared-memory limit: nodes with one cut run in the node kernel, nodes with more
    run on the single-tableau path.  At width 1 the trees fall out of step, so one round carries both kinds."""
    jm = problems.knapsack_mip_model(40, 100, seed=21)
    H, W = Model().loadJson(jm).initial_tableau().matrix.shape
    jm = problems.knapsack_mip_model(40, 100 + max_resident_height(W) - 1 - H, seed=21)
    H, W = Model().loadJson(jm).initial_tableau().matrix.shape
    assert H + 1 == max_resident_height(W)
    got = assert_equals_solve(jm, seeded_cases(jm, 6, seed=4, spread=0.05), width=1)
    assert all(r.get("isIntegral") for r in got)


def test_edge_roots():
    infeasible_root = {"optimize": "v", "opType": "max", "constraints": {"c": {"max": 4}, "d": {"min": 1}},
                       "variables": {"a": {"v": 1, "c": 1, "d": 1}}, "ints": {"a": 1}}
    cases = [{"rhs": {"d": 5}}, {"rhs": {"d": 2.5}}, {"rhs": {"c": 3}}, {"cost": {"a": -1}}]
    assert_equals_solve(infeasible_root, cases)
    unbounded = {"optimize": "v", "opType": "max", "constraints": {"c": {"min": 1}},
                 "variables": {"a": {"v": 1, "c": 1}, "b": {"v": 0, "c": 1}}, "ints": {"a": 1}}
    assert_equals_solve(unbounded, [{"rhs": {"c": 2}}, {"cost": {"a": -1}}, {"cost": {"a": -1, "b": -1}}])
    parity = {"optimize": "v", "opType": "max", "constraints": {"odd": {"equal": 3}},
              "variables": {"a": {"v": 1, "odd": 2}, "b": {"v": 1, "odd": 2}}, "ints": {"a": 1, "b": 1}}
    assert_equals_solve(parity, [{"rhs": {"odd": 4}}, {"rhs": {"odd": 5}}, {}])


def test_cycling_scenario():
    jm = beale_mip()
    assert_equals_solve(jm, [{}, {"rhs": {"r3": 2}}, {"cost": {"x0": -1}}])


def test_continuous_lp_is_its_root():
    jm = {"optimize": "profit", "opType": "max",
          "constraints": {"wood": {"max": 300}, "labor": {"max": 110}, "floor": {"min": 1}},
          "variables": {"table": {"wood": 30, "labor": 5, "profit": 1200, "floor": 1},
                        "dresser": {"wood": 20, "labor": 10, "profit": 1600, "floor": 1}}}
    assert_equals_solve(jm, [{}, {"rhs": {"wood": 200}}, {"rhs": {"floor": 1000}}, {"cost": {"table": 9000}}])


def test_largest_fixture_beyond_shared_memory():
    big = [jm for jm in mip_fixtures() if not small(jm)]
    if not big:
        pytest.skip("no MIP fixture beyond shared memory in the bundle")
    jm = strip_timeouts(min(big, key=lambda m: len(m["variables"])))  # Monster_II
    assert_equals_solve(jm, seeded_cases(jm, 2, seed=1, spread=0.02))

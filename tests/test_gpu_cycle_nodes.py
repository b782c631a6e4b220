"""Branch and cut on MIPs whose node LPs cycle below a clean root, bit for bit against the oracle on every node path
(tests/cycle_models.py; tests/test_cycle_models_cpu.py checks the models on the oracle).

The device stops a cycling node LP by screening its pivot log and solving the node again on the single tableau, where
the reference's stop-before-the-repeat rule is exact: after the node kernel (the whole log, once the CTA ends) and
across the polls of the node slots (two histories per slot, one per phase, carried from poll to poll and reset when
the slot loads a node).  A cycling node is infeasible in the reference; left to itself the device's LP ends feasible a
few turns later, so a redo that does not happen shows in the node log.  Every case compares the whole node log (the
evaluation column of infeasible nodes included), the final tableau, labels, evaluation, flags and Solve()'s result,
and the redo counters of jslp_bnb_status show that the path the case names ran."""
import numpy as np
import pytest

import cycle_models as C
from test_gpu_bnb_state import assert_state, run_and_check, solver

pytestmark = pytest.mark.gpu

CASES = {cid: (jm, cyc) for cid, jm, cyc in C.cases()}
SMALL = ["phase1", "phase2", "prune"]
PADDED = ["phase1_padded", "phase2_padded", "prune_padded"]
OPT_NODE_SLOTS = 10


def counters(b):
    return b.cycle_redos_kernel, b.cycle_redos_slots, b.cycle_redos_pruned


def speculated_cycles(cid, width):
    """Cycling node LPs a round of `width` evaluates: the committed ones, plus (prune models, width >= 3) the cycling
    node that sorts after the integer plan of its round."""
    return len(CASES[cid][1]) + (1 if cid.startswith("prune") and width >= 3 else 0)


@pytest.mark.parametrize("width", [1, 2, 4, 16])
@pytest.mark.parametrize("cid", SMALL)
def test_node_kernel_cycle_hit_redo(cid, width):
    """Engine 4: every node after the root runs in the shared-memory node kernel, which ends the cycling LP inside its
    log; the screen finds the repeat and the node is solved again."""
    jm, _ = CASES[cid]
    b = run_and_check(jm, 0, solver((4, width)), f"{cid} kernel width {width}")
    print(cid, width, counters(b), b.node_kernel_ms)
    assert b.node_kernel_ms > 0 and b.slot_pivots == 0
    assert counters(b) == (speculated_cycles(cid, width), 0, 0), counters(b)


@pytest.mark.parametrize("slots", [1, 2, None])
@pytest.mark.parametrize("steps", [1, 2, 3, None])
@pytest.mark.parametrize("cid", PADDED)
def test_node_slot_cycle_redo(cid, steps, slots):
    """Engine 2, width 16, past shared memory: the nodes of a round run in node slots (one slot is no slot batch:
    every node on the single tableau).  At 1, 2 and 3 steps per poll the repeat spans several polls."""
    jm, cyc = CASES[cid]
    b = run_and_check(jm, 0, solver((2, 16, slots, steps)), f"{cid} slots {slots} steps {steps}")
    print(cid, slots, steps, counters(b), b.slot_pivots)
    assert b.node_kernel_ms == 0
    if slots == 1:
        assert b.slot_pivots == 0 and counters(b) == (0, 0, 0)
        return
    assert b.slot_pivots > 0
    kernel, redone, dropped = counters(b)
    assert kernel == 0 and redone == len(cyc), counters(b)
    # The prune model's round runs (z >= 1, y <= 0), the plan and (z <= 0, y <= 0) side by side when it has three
    # slots or more.  At 32 steps per poll the plan ends in the poll that shows the third node's repeat, so its redo is
    # the one dropped; at fewer steps the plan ends first and the running node is aborted before its repeat shows.
    assert dropped == (1 if cid == "prune_padded" and slots is None and steps is None else 0), counters(b)


@pytest.mark.parametrize("engine", [1, 2])
@pytest.mark.parametrize("cid", SMALL + PADDED)
def test_single_tableau_control(cid, engine):
    """Engines 1 and 2 without node slots: every node on the single tableau, whose own check stops the cycle; no
    screen, no redo."""
    jm, _ = CASES[cid]
    s = solver((engine, 8))
    s.node_slots = 0
    b = run_and_check(jm, 0, s, f"{cid} engine {engine}")
    assert b.node_kernel_ms == 0 and b.slot_pivots == 0 and counters(b) == (0, 0, 0)


def test_two_ranks(tmp_path):
    """Two sharded ranks over gloo: the node kernel (engine 4, every round sharded) and node slots (padded, engine 2).
    Each cycling node is screened and redone on the rank it was dealt to."""
    from oracle import ref_model
    from test_gpu_bnb_state import assert_log_bits
    from test_gpu_dist_edges import assert_identical_ranks, bits, launch, local_solve
    cases = []
    for cid in SMALL:
        cases.append(dict(id=f"kernel_{cid}", model=CASES[cid][0], engine=4, width=16, shard_policy=1, max_nodes=0))
    for cid in PADDED:
        for steps in (2, None):
            cases.append(dict(id=f"slots_{cid}_{steps}", model=CASES[cid][0], engine=2, width=16, shard_policy=1,
                              max_nodes=0, slot_steps=steps))
    res = launch(2, cases, tmp_path)
    failures = []
    for case in cases:
        what = case["id"]
        try:
            ranks = res[what]
            assert_identical_ranks(ranks, what)
            a, m = ranks[0]
            assert m["error"] is None, (what, m["error"])
            osol = ref_model.solve_full(case["model"], fast_cycles=True, node_log=1 << 20)
            assert_log_bits(a["node_log"], osol.tableau.node_log(), what)
            assert m["evaluation"] == float(osol.evaluation).hex(), (what, m["evaluation"], osol.evaluation)
            assert m["result"] == ref_model.simplify(osol), what
            assert np.array_equal(bits(a["matrix"]), bits(osol.tableau.matrix())), what
            assert np.array_equal(a["vrow"], osol.tableau.maps()[0]), what
            assert m["result"] == local_solve(case)[0], what
            st = [mm["status"] for _, mm in ranks]
            key = "cycle_redos_kernel" if what.startswith("kernel") else "cycle_redos_slots"
            assert sum(s[key] for s in st) >= 1, (what, st)
            if what.startswith("slots"):  # a round of two nodes gives each rank one: the infeasible one runs no pivot
                assert any(s["slot_pivots"] > 0 for s in st) and all(s["cycle_redos_kernel"] == 0 for s in st), (what, st)
            else:
                assert all(s["cycle_redos_slots"] == 0 for s in st), (what, st)
        except AssertionError as e:
            failures.append(f"{what}: {e}")
    assert not failures, "\n".join(failures)


def test_bnb_batch_with_a_cycling_tree():
    """jslp_bnb_batch (MIPScenarios' engine) with the phase-1 witness as one of its trees, next to edits whose trees
    do not cycle: every scenario's status is the oracle's for the edited model."""
    from jslpsolver_b200 import mip_scenarios as MS
    from jslpsolver_b200.model import Model
    from oracle import ref_model
    from test_gpu_lp_parity import same_bits
    import jslpsolver_b200 as J
    jm = CASES["phase1"][0]
    specs = [{}, {"rhs": {"Y": 1.5}}, {"rhs": {"d5": 30}}, {"cost": {"u2": 5}}]
    base_m = Model().loadJson(jm)
    base = base_m.initial_tableau()
    edits = [MS.edited(jm, base_m, spec) for spec in specs]
    edges = [MS.edges(base, Model().loadJson(e).initial_tableau()) for e in edits]
    cyc = [ref_model.solve_full(e, fast_cycles=True).state.cyclePhase for e in edits]
    assert cyc[0] == 1
    for width in (1, 8):
        s = J.Solver()
        inst = s._instance(jm, None)
        tab = inst.tableau
        tab.setModel(inst)
        out = tab.bnb_batch(np.array([c for c, _ in edges]), np.array([r for _, r in edges]), width=width)
        tab.close()
        for k, e in enumerate(edits):
            osol = ref_model.solve_full(e, fast_cycles=True)
            got = out["status"][k]
            what = (width, specs[k], cyc[k])
            assert same_bits(got.evaluation, osol.state.evaluation), (what, got.evaluation, osol.state.evaluation)
            assert (got.feasible, got.iterations) == (osol.state.feasible, osol.state.bncIterations), what

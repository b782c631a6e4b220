"""The models of tests/test_gpu_cycle_nodes.py on the oracle alone: each one is what the device file relies on it being,
so that file cannot pass for want of a case.  The root LP is clean and fractional, the nodes that cycle are the ones
named with the phase, length and pivots named, the repeat spans several node-slot polls at the step counts the device
file runs, the cycling LP would end by itself inside the node kernel's log without the check (so the kernel's cycle-hit
redo runs, not its overflow redo), the padded models log the small models' nodes past shared memory, and the prune
models speculate a cycling node behind a better integer plan."""
import numpy as np
import pytest

import cycle_models as C

CASES = {cid: (jm, cyc) for cid, jm, cyc in C.cases()}
NODE_LOG_CAP = 512  # the node kernel's default pivot-log entries per node


def oracle(jm, max_nodes=0):
    from oracle import ref_model
    sol = ref_model.solve_full(jm, fast_cycles=True, node_log=1 << 20, max_nodes=max_nodes)
    assert sol.tableau is not None, jm["name"]
    return sol


@pytest.mark.parametrize("cid", list(CASES))
def test_root_is_clean_and_fractional(cid):
    jm, _ = CASES[cid]
    st = oracle(jm, max_nodes=1).state
    assert st.cyclePhase == 0 and st.feasible and not st.isIntegral
    nl = oracle(jm, max_nodes=1).tableau.node_log()
    assert nl.shape == (1, 8) and nl[0, 2] == 1 and nl[0, 4] == 0 and nl[0, 7] > 0


@pytest.mark.parametrize("cid", list(CASES))
def test_named_nodes_cycle(cid):
    """Replaying every committed node's LP: exactly the named nodes cycle, in the named phase, with the named length
    and pivots; the whole run's cyclePhase (never reset) agrees, and a cycling node is logged infeasible."""
    jm, cyc = CASES[cid]
    sol = oracle(jm)
    nl = sol.tableau.node_log()
    cuts = C.node_cuts(jm)
    assert len(cuts) == len(nl)
    got = {}
    for i, c in enumerate(cuts[1:], 1):  # the root is clean (test above)
        t = C.replay(jm, c)
        st = t.state()
        assert st.lastP1 + st.lastP2 == nl[i, 7], (cid, i)  # the replay is the node the loop ran
        if st.cyclePhase:
            got[i + 1] = (st.cyclePhase, st.cycleLen, st.lastP1, st.lastP2)
    assert got == cyc, (cid, got)
    assert sol.state.cyclePhase == max(p for p, *_ in cyc.values())
    for node in cyc:
        assert nl[node - 1, 2] == 0


@pytest.mark.parametrize("cid", list(CASES))
def test_cycle_spans_several_slot_polls(cid):
    """At the spanning step counts a node slot executes fewer pivots per poll than one turn of the cycle, so the host's
    per-slot histories must carry the repeat from poll to poll."""
    _, cyc = CASES[cid]
    for phase, length, p1, p2 in cyc.values():
        assert all(length > s for s in C.SPANNING_STEPS)
        assert p1 + p2 > 2 * max(C.SPANNING_STEPS)


@pytest.mark.parametrize("cid", list(CASES))
def test_cycling_lp_ends_by_itself_inside_the_node_log(cid):
    """Without the check the cycling node LP leaves the cycle after a few turns (rounding breaks a tie) and ends well
    inside the node kernel's pivot log: the kernel finishes the node, and only the screen of its log sends it back."""
    jm, cyc = CASES[cid]
    cuts = C.node_cuts(jm)
    for node, (phase, length, p1, p2) in cyc.items():
        t = C.replay(jm, cuts[node - 1], check_cycles=False, pivot_limit=4 * NODE_LOG_CAP)
        st = t.state()
        assert not t.truncated() and st.cyclePhase == 0, (cid, node)
        assert p1 + p2 < st.lastP1 + st.lastP2 < NODE_LOG_CAP - 2, (cid, node, st.lastP1, st.lastP2)
        assert st.feasible  # the device's own answer would differ from the reference's: infeasible


@pytest.mark.parametrize("small,padded", [("phase1", "phase1_padded"), ("phase2", "phase2_padded"),
                                          ("prune", "prune_padded")])
def test_padded_model_logs_the_small_models_nodes(small, padded):
    """Every column of the node log is the small model's but the branching variable's element index, which the padding
    rows shift: the variable itself is the same.  Result and solution are the same too."""
    from oracle import ref_model
    a, b = oracle(CASES[small][0]), oracle(CASES[padded][0])
    na, nb = a.tableau.node_log(), b.tableau.node_log()
    assert na.shape == nb.shape
    cols = [0, 1, 2, 3, 4, 6, 7]
    assert np.array_equal(na[:, cols].view(np.uint64), nb[:, cols].view(np.uint64))
    name = lambda sol, i: sol.model.variablesPerIndex[int(i)].id if i >= 0 else None
    assert [name(a, i) for i in na[:, 5]] == [name(b, i) for i in nb[:, 5]]
    assert ref_model.simplify(a) == ref_model.simplify(b)


@pytest.mark.parametrize("cid", ["phase1_padded", "phase2_padded", "prune_padded"])
def test_padded_models_are_past_shared_memory(cid):
    from jslpsolver_b200.model import Model
    H, W = Model().loadJson(CASES[cid][0]).initial_tableau().matrix.shape
    assert H > C.PAD and W > C.PAD and 8 * H * W > 227 * 1024


@pytest.mark.parametrize("cid", ["prune", "prune_padded"])
def test_prune_model_speculates_a_cycling_node_behind_a_better_plan(cid):
    """Commit order: root, z <= 0, z >= 1, (z >= 1, y <= 0) cycling, (z >= 1, y >= 1) integral at -3.5; then the
    frontier holds (z <= 0, y <= 0) and (z <= 0, y >= 1) at relaxed -3 > -3.5, which the reference skips.  A round of
    width 3 or more takes the cycling (z <= 0, y <= 0) after the plan, so its redo must be dropped."""
    from oracle import ref_model
    jm, _ = CASES[cid]
    sol = oracle(jm)
    nl = sol.tableau.node_log()
    assert nl[:, 3].tolist() == [-5.0, -3.0, -4.5, -4.5, -3.5] and nl[4, 4] == 1
    assert ref_model.simplify(sol)["result"] == -3.5
    m = sol.model
    z, y = (next(v.index for v in m.variables if v.id == n) for n in ("z", "y"))
    skipped = [(1, z, 0.0), (1, y, 0.0)]
    assert [tuple(c) for c in C.node_cuts(jm)[1]] == [(1, z, 0.0)]
    t = C.replay(jm, skipped)
    assert t.state().cyclePhase == 1 and t.state().cycleLen == 6
    assert -3.0 > nl[4, 3]  # its relaxed value (its parent's) is worse than the plan's

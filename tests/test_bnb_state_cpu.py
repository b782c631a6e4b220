"""The models of tests/test_gpu_bnb_state.py on the oracle alone: each one is what the device file relies on it being, so
that file cannot pass for want of a case.  Every model must reach branch and cut (not be decided by presolve), the
no-plan models must end without an integer plan, and the node logs must hold infeasible nodes whose evaluation column
would change if a node speculated after them wrote the tableau's evaluation first, at every width the device runs."""
import numpy as np
import pytest

import bnb_state_models as B


def oracle(jm, max_nodes=0):
    from oracle import ref_model
    sol = ref_model.solve_full(jm, fast_cycles=True, node_log=1 << 20, max_nodes=max_nodes)
    assert sol.tableau is not None, jm["name"]
    return sol


@pytest.mark.parametrize("high_fractional", [False, True])
def test_leak_model_values(high_fractional):
    """The hand-worked case: capped at 2 nodes the oracle commits the root and its infeasible low child, keeps the root's
    evaluation in row 2 and as the result; the high child (committed third) has a different evaluation."""
    from oracle import ref_model
    jm = B.leak_model(high_fractional)
    root = 1.0 if high_fractional else 0.5
    sol = oracle(jm, max_nodes=2)
    nl = sol.tableau.node_log()
    assert nl.shape == (2, 8)
    assert nl[0, 2] == 1 and nl[0, 3] == root and nl[0, 4] == 0
    assert nl[1, 2] == 0 and nl[1, 3] == root and nl[1, 1] == 1
    res = ref_model.simplify(sol)
    assert res["feasible"] is False and res["result"] == root
    full = oracle(jm).tableau.node_log()
    assert full[2, 2] == 1 and full[2, 3] == (1.75 if high_fractional else 1.0)
    assert full[2, 4] == (0 if high_fractional else 1)
    assert all(1 in B.leaks(full, w) for w in B.WIDTHS)


@pytest.mark.parametrize("cid", ["parity_small", "parity_capped", "parity_padded"])
def test_parity_models_have_no_integer_plan(cid):
    jm = dict((c, m) for c, m, _ in B.cases())[cid]
    sol = oracle(jm, max_nodes=2003)
    nl = sol.tableau.node_log()
    assert not sol.feasible and not sol.state.isIntegral
    assert nl[0, 2] == 1 and not (nl[:, 4] == 1).any()
    assert (nl[:, 2] == 0).sum() > 10
    if cid == "parity_small":
        assert len(nl) <= 200  # the whole tree
    else:
        assert len(nl) == 2003  # the same tree in both: the padding never binds
    for w in B.WIDTHS:
        assert B.leaks(nl, w), (cid, w)


def test_padded_parity_is_past_shared_memory():
    """At 309 x 307 fp64 a node tableau (740 KB) is far past one SM's 227 KB of shared memory: nodes go to node slots or
    the single-tableau path, never the node kernel."""
    from jslpsolver_b200.model import Model
    H, W = Model().loadJson(B.PADDED_PARITY).initial_tableau().matrix.shape
    assert (H, W) == (309, 307) and 8 * H * W > 227 * 1024


def test_caps_stop_right_after_a_leaking_infeasible_commit():
    caps = dict((c, k) for c, _, k in B.cases())["parity_capped"]
    full = oracle(B.CAPPED_PARITY, max_nodes=2003).tableau.node_log()
    leak4 = B.leaks(full, 4)
    stops = [c for c in caps if c - 1 in leak4]
    assert len(stops) >= 3, caps
    assert any(full[c - 1, 2] == 1 for c in caps), caps  # and one stop after a feasible commit
    for c in caps:
        sol = oracle(B.CAPPED_PARITY, max_nodes=c)
        nl = sol.tableau.node_log()
        assert np.array_equal(nl, full[:c]), c
        assert sol.state.evaluation == nl[-1, 3], c  # the result is the last row's evaluation


def test_root_infeasible_model():
    """The root LP runs phase-1 pivots and ends infeasible: one row, column 3 the evaluation before any LP (0)."""
    sol = oracle(B.root_infeasible_mip())
    nl = sol.tableau.node_log()
    assert nl.shape == (1, 8) and nl[0, 2] == 0 and nl[0, 7] > 0
    assert np.float64(nl[0, 3]).tobytes() == np.float64(0.0).tobytes()
    assert not sol.feasible and sol.state.bncIterations == 1

"""The tableau's evaluation across branch and cut, bit for bit against the oracle on every node path
(tests/bnb_state_models.py; tests/test_bnb_state_cpu.py checks the models' preconditions on the oracle).

The reference logs an infeasible node with the evaluation the tableau kept from the last node that set one, and an
infeasible last node leaves that value as Solve()'s result.  The device evaluates the nodes of a round before it commits
them, some in place on the single tableau, so a node solved ahead of its commit must not leave its evaluation behind.
Every case compares all eight columns of the node log (column 3 of infeasible nodes included), the bits of the final
evaluation, Solve()'s result, flags, final tableau and labels, on the leak cases, models without an integer plan (whole,
capped just after infeasible commits, and past shared memory) and a root that is infeasible, in every branch-and-cut
mode of the suite, engine 1, useMIRCuts, the enhanced and incremental services, a MIP start, two sharded ranks on the
single-tableau and slot paths, and jslp_bnb_batch."""
import numpy as np
import pytest

import bnb_state_models as B
from test_gpu_lp_parity import BNB_MODES, ENHANCED, same_bits, solve_capped

pytestmark = pytest.mark.gpu

CASES = B.cases()
RUNS = [(cid, jm, cap) for cid, jm, caps in CASES for cap in caps]
# the suite's modes, engine 1 and useMIRCuts: (engine, width[, node slots, slot steps[, tab options]]), model options
MODES = {name: (spec, {}) for name, spec in BNB_MODES.items()}
MODES["engine1_spec8"] = ((1, 8), {})
MODES["mir_spec8"] = ((0, 8), {"useMIRCuts": True})


def solver(spec):
    import jslpsolver_b200 as J
    s = J.Solver()
    s.engine, s.max_spec_batch = spec[:2]
    if len(spec) > 2:
        s.node_slots, s.slot_steps = spec[2:4]
    if len(spec) > 4:
        s.options = dict(spec[4])
    return s


def with_options(jm, opts):
    return dict(jm, options=dict(jm.get("options") or {}, **opts)) if opts else jm


def assert_log_bits(gnl, onl, what):
    assert gnl.shape == onl.shape, (what, gnl.shape, onl.shape)
    for i in range(len(onl)):
        assert same_bits(gnl[i], onl[i]), f"{what} node {i}: gpu={gnl[i].tolist()} oracle={onl[i].tolist()}"


def assert_state(s, gsol, osol, what):
    """Node log, evaluation bits, Solve()'s dict, flags, final tableau and labels."""
    from oracle import ref_model
    gt, ot = gsol._tableau, osol.tableau
    assert_log_bits(gt.node_log(), ot.node_log(), what)
    st = osol.state
    assert same_bits(gt.evaluation, st.evaluation), (what, gt.evaluation, st.evaluation)
    assert s._simplified(gsol) == ref_model.simplify(osol), (what, s._simplified(gsol), ref_model.simplify(osol))
    assert gt.branchAndCutIterations == st.bncIterations, what
    assert (gt.feasible, gt.bounded) == (bool(st.feasible), bool(st.bounded)), what
    assert same_bits(gt.matrix2d(), ot.matrix()), what
    assert np.array_equal(gt.varIndexByRow, ot.maps()[0]) and np.array_equal(gt.varIndexByCol, ot.maps()[1]), what


def run_and_check(jm, cap, s, what):
    from oracle import ref_model
    osol = ref_model.solve_full(jm, fast_cycles=True, node_log=1 << 20, max_nodes=cap)
    assert osol.tableau is not None, what
    gsol = solve_capped(s, jm, cap)
    assert_state(s, gsol, osol, what)
    return gsol._tableau.lastBnbStatus


def backend(cid, mode, b):
    """Where a case's nodes must have run: the node kernel (automatic engine, nodes that fit), node slots (padded
    model, slot modes) or one after another on the single tableau."""
    print(f"{cid} {mode}: nodes {b.iterations} node kernel {b.node_kernel_ms:.3f} ms slot pivots {b.slot_pivots}")
    if mode in ("hbm_seq", "hbm_noslots_spec4", "engine1_spec8", "mir_spec8"):
        assert b.node_kernel_ms == 0 and b.slot_pivots == 0, (cid, mode)
    elif cid == "parity_padded" and mode in ("hbm_spec4", "hbm_slots3_steps5", "auto_spec8", "auto_spec32"):
        assert b.node_kernel_ms == 0 and b.slot_pivots > 0, (cid, mode)
    elif cid in ("parity_small", "parity_capped") and mode.startswith("auto"):
        assert b.node_kernel_ms > 0, (cid, mode)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("run", RUNS, ids=lambda r: f"{r[0]}-cap{r[2]}")
def test_every_mode_matches_the_oracle(run, mode):
    cid, jm, cap = run
    spec, opts = MODES[mode]
    b = run_and_check(with_options(jm, opts), cap, solver(spec), f"{cid} cap {cap} {mode}")
    if cap != 2:  # two nodes: the root and one child, no speculated round to speak of
        backend(cid, mode, b)


@pytest.mark.parametrize("mode", ["hbm_seq", "hbm_noslots_spec4", "auto_spec8_logcap3", "engine1_spec8"])
@pytest.mark.parametrize("high_fractional", [False, True])
def test_leak_case_written_out(high_fractional, mode):
    """The hand-worked case, capped at two nodes: the root and its infeasible low child are committed, the high child
    (evaluated in the same round at width >= 2) is not.  Row 2 and the result keep the root's evaluation.  (Under
    useMIRCuts the root's cuts make it integral: the parity models carry that mode.)"""
    spec, opts = MODES[mode]
    s = solver(spec)
    gsol = solve_capped(s, with_options(B.leak_model(high_fractional), opts), 2)
    root = 1.0 if high_fractional else 0.5
    nl = gsol._tableau.node_log()
    assert nl.shape == (2, 8) and nl[1, 2] == 0 and same_bits(nl[1, 3], root), nl.tolist()
    res = s._simplified(gsol)
    assert res["feasible"] is False and same_bits(res["result"], root), res


@pytest.mark.parametrize("opts", [ENHANCED[0], ENHANCED[4]], ids=["enhanced", "incremental"])
@pytest.mark.parametrize("run", RUNS, ids=lambda r: f"{r[0]}-cap{r[2]}")
def test_services_match_the_oracle(run, opts):
    import jslpsolver_b200 as J
    cid, jm, cap = run
    if cid == "parity_padded":
        pytest.skip("the services evaluate one node at a time: the small models cover them")
    run_and_check(with_options(jm, opts), cap, J.Solver(), f"{cid} cap {cap} {opts}")


@pytest.mark.parametrize("engine,width,slots", [(2, 8, 0), (0, 8, None), (2, 1, None)])
def test_mip_start_on_a_model_without_a_plan(engine, width, slots):
    """The seed stage runs its dives through the round evaluator; no start completes, so the tree and every logged
    evaluation are those of the plain loop."""
    import mip_start_oracle as MSO
    from test_gpu_mip_start import run
    for cap in dict((c, k) for c, _, k in CASES)["parity_capped"][:2]:
        jm = B.CAPPED_PARITY
        start = [{"x0": None, "x1": 1}, {k: None for k in jm["variables"]}]
        simp, report, res = MSO.solve(jm, start, max_nodes=cap)
        m, sol, simplified = run(jm, start, width=width, engine=engine, slots=slots, max_nodes=cap)
        t = m.tableau
        what = f"start cap {cap} engine {engine} width {width}"
        assert_log_bits(t.node_log(), res["node_log"], what)
        assert same_bits(t.lastBnbStatus.evaluation, res["o"].state().evaluation), what
        assert simplified == simp and sol.mipStart == report, what
        assert [g.status for g in t.lastStartStatus] == [o["status"] for o in res["starts"]], what


def test_bnb_batch_on_models_without_a_plan():
    """jslp_bnb_batch keeps each tree's evaluation in its own scalars: every scenario's status.evaluation is the oracle's
    for the edited model, whole and capped."""
    from jslpsolver_b200 import mip_scenarios as MS
    from jslpsolver_b200.model import Model
    from oracle import ref_model
    import jslpsolver_b200 as J
    for jm in (B.SMALL_PARITY, B.CAPPED_PARITY):
        odd = jm["constraints"]["odd"]["equal"]
        specs = [{}, {"rhs": {"odd": odd + 2}}, {"rhs": {"odd": odd - 1}}, {"cost": {"x0": 0.5}}]
        base_m = Model().loadJson(dict(jm, options={"presolve": False}))
        base = base_m.initial_tableau()
        edits = [MS.edited(jm, base_m, spec) for spec in specs]
        edges = [MS.edges(base, Model().loadJson(e).initial_tableau()) for e in edits]
        for cap in (0, 21, 23, 60) if jm is B.CAPPED_PARITY else (0, 40):
            if jm is B.CAPPED_PARITY and cap == 0:
                continue
            for width in (1, 8):
                s = J.Solver()
                inst = s._instance(dict(jm, options={"presolve": False}), None)
                tab = inst.tableau
                tab.setModel(inst)
                out = tab.bnb_batch(np.array([c for c, _ in edges]), np.array([r for _, r in edges]), max_nodes=cap,
                                    width=width)
                tab.close()
                for k, e in enumerate(edits):
                    osol = ref_model.solve_full(e, fast_cycles=True, max_nodes=cap)
                    got = out["status"][k]
                    what = (jm["name"], cap, width, specs[k])
                    assert same_bits(got.evaluation, osol.state.evaluation), (what, got.evaluation, osol.state.evaluation)
                    assert (got.feasible, got.iterations) == (osol.state.feasible, osol.state.bncIterations), what


# ------------------------------------------------------------------ two ranks (tests/dist_edges_worker.py)
OPT_NODE_SLOTS = 10


def sharded_cases():
    cases = []
    for cid, jm, caps in CASES:
        if cid == "root_infeasible":
            continue
        for cap in caps:
            if cid == "parity_padded":  # engine 2 with node slots
                cases.append(dict(id=f"w2_slots_{cid}_{cap}", model=jm, engine=2, width=8, shard_policy=1, max_nodes=cap))
            else:  # engine 2 without slots: every node on the single tableau
                cases.append(dict(id=f"w2_single_{cid}_{cap}", model=jm, engine=2, width=4, shard_policy=1,
                                  max_nodes=cap, options={OPT_NODE_SLOTS: 0}))
    return cases


def test_two_ranks_match_the_oracle(tmp_path):
    from oracle import ref_model
    from test_gpu_dist_edges import assert_identical_ranks, bits, launch, local_solve
    cases = sharded_cases()
    res = launch(2, cases, tmp_path)
    failures = []
    for case in cases:
        what = case["id"]
        try:
            ranks = res[what]
            assert_identical_ranks(ranks, what)
            a, m = ranks[0]
            assert m["error"] is None, (what, m["error"])
            osol = ref_model.solve_full(case["model"], fast_cycles=True, node_log=1 << 20, max_nodes=case["max_nodes"])
            assert_log_bits(a["node_log"], osol.tableau.node_log(), what)
            assert m["evaluation"] == float(osol.evaluation).hex(), (what, m["evaluation"], osol.evaluation)
            assert m["result"] == ref_model.simplify(osol), what
            assert np.array_equal(bits(a["matrix"]), bits(osol.tableau.matrix())), what
            assert np.array_equal(a["vrow"], osol.tableau.maps()[0]), what
            assert m["result"] == local_solve(case)[0], what
            st = [mm["status"] for _, mm in ranks]
            assert st[0]["collectives"] >= st[0]["rounds"] - 1 > 0, (what, st[0])
            if "slots" in what:
                assert all(s["slot_pivots"] > 0 for s in st), (what, st)
            else:
                assert all(s["slot_pivots"] == 0 and s["node_kernel_ms"] == 0 for s in st), (what, st)
        except AssertionError as e:
            failures.append(f"{what}: {e}")
    assert not failures, "\n".join(failures)

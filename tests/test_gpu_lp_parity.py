"""GPU parity tests: the CUDA path (through the C ABI) against the oracle on the same inputs.
Bit-exact for everything integer (flags, pivot sequence, basis index arrays) AND for the fp64
tableau itself: both sides perform the same IEEE operations in the same order per element, so
the whole matrix must be identical, not merely close (the north_star's 1e-9 is the outer bar)."""
import numpy as np
import pytest

from conftest import load_bundle
from helpers import compare_solutions, strip_timeouts

pytestmark = pytest.mark.gpu
BUNDLE = load_bundle()
# engine, or (engine, look-ahead tail on/off, fused-step kernel variant)
ENGINES = {"two_kernel": 1, "fused": 2, "resident": 4, "fused_generic_tail": (2, 0, 0),
           "fused_v1_prefetch": (2, 1, 1), "fused_v2_occ4": (2, 1, 2), "fused_v3_t512": (2, 1, 3),
           "fused_v5_t128": (2, 1, 5), "fused_pdl": (2, 1, 0, 1), "fused_generic_pdl": (2, 0, 3, 1),
           "fused_inplace": (2, 1, 0, 0, 0), "fused_inplace_v3": (2, 1, 3, 0, 0)}


def same_bits(a, b):
    """Bit for bit: -0.0 differs from +0.0 (JS sees the sign through 1 / x and Math.min), any NaN equals any NaN (JS
    cannot observe a NaN's payload)."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    if a.shape != b.shape:
        return False
    return bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


def oracle_lp(it, precision=1e-8, check_cycles=True, log=1 << 16):
    from oracle import ref_model
    t = ref_model.OracleTableau(it.matrix, it.varIndexByRow, it.varIndexByCol, precision=precision,
                                unrestricted=it.unrestricted, integers=it.integerIndices,
                                opt_rc=it.optionalCosts, check_cycles=check_cycles, fast_cycles=True,
                                pivot_log=log)
    return t


def gpu_lp(it, engine, precision=1e-8, batch=None, log=1 << 16, grid_per_sm=None, timeline=None):
    """engine: JSLP_OPT_ENGINE value, or a tuple (engine, lookahead, step variant[, PDL[, ping-pong]]).
    grid_per_sm: JSLP_OPT_GRID_PER_SM (step CTAs per SM); timeline: JSLP_OPT_TIMELINE (pivot steps recorded)."""
    from jslpsolver_b200 import _lib
    from jslpsolver_b200.tableau import GpuTableau
    lookahead = variant = pdl = pingpong = None
    if isinstance(engine, tuple):
        spec = engine
        engine, lookahead, variant = spec[:3]
        pdl = spec[3] if len(spec) > 3 else None
        pingpong = spec[4] if len(spec) > 4 else None
    g = GpuTableau(precision)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, it.integerIndices, it.optionalCosts)
    g.set_option(_lib.OPT_ENGINE, engine)
    g.set_option(_lib.OPT_PIVOT_LOG_CAP, log)
    if lookahead is not None:
        g.set_option(_lib.OPT_LOOKAHEAD, lookahead)
    if variant is not None:
        g.set_option(_lib.OPT_STEP_VARIANT, variant)
    if pdl is not None:
        g.set_option(_lib.OPT_PDL, pdl)
    if pingpong is not None:
        g.set_option(_lib.OPT_PINGPONG, pingpong)
    if batch:
        g.set_option(_lib.OPT_BATCH, batch)
    if grid_per_sm is not None:
        g.set_option(_lib.OPT_GRID_PER_SM, grid_per_sm)
    if timeline is not None:
        g.set_option(_lib.OPT_TIMELINE, timeline)
    return g


def assert_lp_parity(g, o, what=""):
    st, os_ = g.lastStatus, o.state()
    glog, olog = g.pivot_log(), o.pivot_log()
    n = min(len(glog), len(olog))
    if not np.array_equal(glog[:n], olog[:n]) or len(glog) != len(olog):
        first = next((i for i in range(n) if not np.array_equal(glog[i], olog[i])), n)
        raise AssertionError(f"{what}: pivot sequence differs at pivot {first}: gpu={glog[first:first+3].tolist()} "
                             f"oracle={olog[first:first+3].tolist()} (lengths {len(glog)} vs {len(olog)})")
    assert (bool(st.feasible), bool(st.bounded)) == (bool(os_.feasible), bool(os_.bounded)), what
    assert (st.phase1_pivots, st.phase2_pivots) == (os_.lastP1, os_.lastP2), what
    assert st.cycled == os_.cyclePhase, what
    if st.cycled:
        assert (st.cycle_start, st.cycle_length) == (os_.cycleStart, os_.cycleLen), what
    vr, vc = o.maps()
    assert np.array_equal(g.varIndexByRow, vr) and np.array_equal(g.varIndexByCol, vc), what
    assert same_bits(g.matrix2d(), o.matrix()), f"{what}: tableau bits differ"
    if st.feasible and st.bounded and not st.cycled:
        assert same_bits(st.evaluation, os_.evaluation), what
    if g.nOpt:
        assert same_bits(g.optional_reduced_costs(), o.optional()), what


def assert_node_log_parity(gt, ot, what=""):
    """Branch-and-cut node logs of the device tableau gt and the oracle tableau ot: same nodes in the same order, same
    integer fields, and the bits of the branching value and the evaluation (an infeasible node logs the evaluation the
    tableau kept from the last node that set one)."""
    onl, gnl = ot.node_log(), gt.node_log()
    assert gnl.shape == onl.shape, (what, gnl.shape, onl.shape)
    for i in range(len(onl)):
        a, b = gnl[i], onl[i]
        ok = all(a[k] == b[k] for k in (0, 1, 2, 4, 5, 7)) and same_bits(a[6], b[6]) and same_bits(a[3], b[3])
        assert ok, f"{what} node {i}: gpu={a.tolist()} oracle={b.tolist()}"


# ------------------------------------------------------------------ golden fixtures end to end
@pytest.mark.parametrize("fx", BUNDLE["fixtures"] + BUNDLE["readme"], ids=lambda f: f["file"])
def test_fixture_solve_matches_reference_expects_and_oracle(fx):
    import jslpsolver_b200 as J
    from oracle import ref_model
    jm = strip_timeouts(fx["model"])
    res = J.Solve(jm)
    bad = compare_solutions(res, fx["expects"])
    assert not bad, bad
    ores = ref_model.Solve(jm, fast_cycles=True)
    assert list(res.keys()) == list(ores.keys()), (res, ores)
    for k in res:
        assert res[k] == ores[k] or (res[k] != res[k] and ores[k] != ores[k]), (k, res[k], ores[k])


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("fx", [f for f in BUNDLE["fixtures"] if not (f["model"].get("ints") or f["model"].get("binaries"))],
                         ids=lambda f: f["file"])
def test_lp_fixture_tableau_bits(fx, engine):
    """Continuous fixtures: pivot sequence, basis arrays, flags and every tableau bit."""
    import jslpsolver_b200.tableau as T
    from jslpsolver_b200.model import Model, presolve
    jm = strip_timeouts(fx["model"])
    m = Model().loadJson(jm)
    if m.usePresolve:
        pr = presolve(m)
        if pr.isInfeasible:
            pytest.skip("decided by presolve")
        for v in pr.fixedVariables:
            v.cost = 0
    it = m.initial_tableau()
    o = oracle_lp(it, check_cycles=m.checkForCycles)
    o.simplex()
    g = gpu_lp(it, ENGINES[engine])
    g.model = m
    g.simplex()
    assert_lp_parity(g, o, fx["file"])


# ------------------------------------------------------------------ seeded dense LPs
@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("n,m,seed", [(5, 4, 1), (30, 20, 2), (64, 64, 3), (150, 120, 4), (333, 257, 5), (600, 500, 6)])
def test_dense_packing_lp(n, m, seed, engine):
    from jslpsolver_b200 import problems
    it = problems.dense_packing_lp_tableau(n, m, seed)
    o = oracle_lp(it)
    o.simplex()
    g = gpu_lp(it, ENGINES[engine])
    g.simplex()
    assert_lp_parity(g, o, f"dense {n}x{m}")
    assert g.lastStatus.phase2_pivots > 0


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("n,m,seed", [(12, 9, 11), (40, 30, 12), (120, 80, 13), (260, 200, 14)])
def test_mixed_lp_with_phase1(n, m, seed, engine, monkeypatch):
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    mod = Model().loadJson(problems.mixed_lp_model(n, m, seed))
    it = mod.initial_tableau()
    o = oracle_lp(it)
    o.simplex()
    g = gpu_lp(it, ENGINES[engine])
    g.simplex()
    assert_lp_parity(g, o, f"mixed {n}x{m}")


@pytest.mark.parametrize("engine", ["auto", "fused_inplace"])
def test_wide_mixed_lp_with_phase1(engine):
    """31 x 2101 tableau: the row stride (2112) exceeds 8 columns x 256 threads, so the ping-pong selector derives the
    phase-1 entering column with the wide-tableau loop instead of its register-resident fast path."""
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    it = Model().loadJson(problems.mixed_lp_model(2100, 30, seed=15)).initial_tableau()
    o = oracle_lp(it)
    o.simplex()
    g = gpu_lp(it, 0 if engine == "auto" else ENGINES[engine])
    g.simplex()
    assert_lp_parity(g, o, f"wide mixed 2100x30 {engine}")
    assert g.lastStatus.phase1_pivots > 0


@pytest.mark.parametrize("batch", [1, 2, 3, 7])
def test_small_batches_and_cycle_rewind(batch):
    """Cycle detection runs on the host over the drained log; with tiny batches the rewind
    (snapshot + replay to the pivot before the repeat) is exercised at every offset."""
    from jslpsolver_b200.model import Model
    names = {"Cycling Fletcher.json", "Cycling introductory example.json", "Degenerate Max.json",
             "Cycling steepest edge column selection.json", "Monster Problem.json"}
    for fx in BUNDLE["fixtures"]:
        if fx["file"] not in names:
            continue
        m = Model().loadJson(strip_timeouts(fx["model"]))
        it = m.initial_tableau()
        o = oracle_lp(it, check_cycles=m.checkForCycles)
        o.simplex()
        g = gpu_lp(it, 2, batch=batch)
        g.model = m
        g.simplex()
        assert_lp_parity(g, o, f"{fx['file']} batch={batch}")


def test_forced_cycle_is_detected_like_the_reference():
    """Beale-type cycling LP under Dantzig + lowest-index ratio rule; whatever the reference
    rules do with it (cycle or not), flags, counts and the stopping tableau must agree."""
    from jslpsolver_b200.model import Model
    model = {"optimize": "z", "opType": "max",
             "constraints": {"c1": {"max": 0}, "c2": {"max": 0}, "c3": {"max": 1}},
             "variables": {"x1": {"z": 0.75, "c1": 0.25, "c2": 0.5},
                           "x2": {"z": -150, "c1": -60, "c2": -90},
                           "x3": {"z": 0.02, "c1": -0.04, "c2": -0.02, "c3": 1},
                           "x4": {"z": -6, "c1": 9, "c2": 3}}}
    m = Model().loadJson(model)
    it = m.initial_tableau()
    for batch in (1, 2, 5, 256):
        o = oracle_lp(it)
        o.simplex()
        g = gpu_lp(it, 2, batch=batch)
        g.simplex()
        assert_lp_parity(g, o, f"beale batch={batch}")


# ------------------------------------------------------------------ seam primitives
def test_pivot_save_restore_cuts_and_mip_scan():
    from jslpsolver_b200 import problems
    it = problems.dense_packing_lp_tableau(23, 17, seed=9)
    ints = np.array([17 + j for j in range(0, 23, 2)], dtype=np.int32)
    it.integerIndices = ints
    o = oracle_lp(it)
    g = gpu_lp(it, 2)
    for (r, c) in [(3, 4), (7, 1), (1, 23), (17, 12)]:
        o.pivot(r, c)
        g.pivot(r, c)
    assert same_bits(g.matrix2d(), o.matrix())
    assert np.array_equal(g.varIndexByRow, o.maps()[0]) and np.array_equal(g.varIndexByCol, o.maps()[1])
    o.simplex(); g.simplex()
    assert_lp_parity(g, o, "after explicit pivots")
    assert g.isIntegral() == o.is_integral()
    iv, val = o.most_fractional()
    mf = g.getMostFractionalVar()
    assert (mf["index"] if mf["index"] is not None else -1) == iv and same_bits(mf["value"], val)
    o.save(); g.save()
    basic = int(o.maps()[0][2])          # a basic variable
    nonbasic = int(o.maps()[1][3])       # a non-basic variable
    cuts = [("min", basic, 1.0), ("max", nonbasic, 2.0), ("max", basic, 5.0)]
    o.add_cuts(cuts); g.addCutConstraints(cuts)
    assert g.height == o.state().height
    assert same_bits(g.matrix2d(), o.matrix())
    assert np.array_equal(g.varIndexByRow, o.maps()[0])
    o.simplex(); g.simplex()
    assert_lp_parity(g, o, "after cuts")
    o.restore(); g.restore()
    assert g.height == o.state().height and same_bits(g.matrix2d(), o.matrix())
    st = o.apply_cuts(cuts[:2]); g.applyCuts(cuts[:2])
    assert_lp_parity(g, o, "applyCuts")


def test_row_capacity_growth():
    from jslpsolver_b200 import problems
    from jslpsolver_b200.tableau import GpuTableau
    it = problems.dense_packing_lp_tableau(9, 6, seed=21)
    o = oracle_lp(it)
    g = GpuTableau(1e-8)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, row_capacity=7)
    o.simplex(); g.simplex()
    o.save(); g.save()
    nb = [int(v) for v in o.maps()[1][1:6]]
    cuts = [("max", v, 3.0) for v in nb] * 5
    o.add_cuts(cuts); g.addCutConstraints(cuts)
    assert same_bits(g.matrix2d(), o.matrix())
    o.simplex(); g.simplex()
    assert same_bits(g.matrix2d(), o.matrix())


# ------------------------------------------------------------------ branch and cut
# (engine, speculation width): HBM path one node at a time (the reference's literal order), then
# speculative rounds with shared-memory-resident node batches
# (engine, speculation width[, node slots, pivots per slot per poll]): "hbm_spec4" runs its rounds in HBM node
# slots (K3, jslp_slots.cuh), the two "slots" modes force odd slot counts / tiny poll windows
BNB_MODES = {"hbm_seq": (2, 1), "auto_seq": (0, 1), "auto_spec8": (0, 8), "auto_spec32": (0, 32), "hbm_spec4": (2, 4),
             "hbm_slots3_steps5": (2, 16, 3, 5), "hbm_noslots_spec4": (2, 4, 0, 32),
             # shared-memory node kernel with a 3-entry pivot log: every node that needs more overflows and is
             # re-evaluated on the HBM path (the boundary of jslp_bnb.cuh's log_cap / max_pivots handling)
             "auto_spec8_logcap3": (0, 8, None, None, {14: 3})}


def _generated_mips():
    """Branch-and-cut inputs built by problems.half_tie_mip_model, in the shape of a fixture: the LP relaxation keeps
    most basic integer variables at exactly k + 1/2, so the position tie-break picks the branching variable at nearly
    every node.  80 integer rows (the root and its nodes fit the shared-memory node kernel, integer rows in three
    warps) and 300 (past one 256-thread pass of the MIP scan; the HBM path and node slots).  max_nodes caps the loop."""
    from jslpsolver_b200 import problems
    return [{"file": f"half_tie_{n}", "model": problems.half_tie_mip_model(n, seed=n), "max_nodes": cap, "k2": n == 80}
            for n, cap in ((80, 120), (300, 40))]


GENERATED_MIPS = _generated_mips()
MIP_FIXTURES = [f for f in BUNDLE["fixtures"] if (f["model"].get("ints") or f["model"].get("binaries"))]
GENERATED_MODES = ("hbm_seq", "auto_spec8", "hbm_spec4", "hbm_slots3_steps5", "auto_spec8_logcap3")


def solve_capped(s, jm, max_nodes=0):
    """s.Solve(jm, full=True) with the branch-and-cut loop stopped after max_nodes nodes (0 = no cap)."""
    inst = s._instance(jm, None)
    inst.max_nodes = max_nodes
    return s._finish(inst, inst.solve(), True)


def assert_backend(gt, fx, mode):
    """A generated MIP reached the back end its mode names: the shared-memory node kernel (automatic engine, nodes
    that fit), node slots (speculated rounds of nodes that do not, or engine 2), or neither (one node at a time)."""
    b = gt.lastBnbStatus
    print(f"{fx['file']} {mode}: nodes {b.iterations} node kernel {b.node_kernel_ms:.3f} ms slot pivots {b.slot_pivots}")
    if mode == "hbm_seq":
        assert b.node_kernel_ms == 0 and b.slot_pivots == 0, (mode, b.node_kernel_ms, b.slot_pivots)
    elif mode.startswith("auto") and fx["k2"]:
        assert b.node_kernel_ms > 0, (mode, b.node_kernel_ms)
    else:
        assert b.node_kernel_ms == 0 and b.slot_pivots > 0, (mode, b.node_kernel_ms, b.slot_pivots)


@pytest.mark.parametrize("mode", list(BNB_MODES))
@pytest.mark.parametrize("fx", MIP_FIXTURES + GENERATED_MIPS, ids=lambda f: f["file"])
def test_mip_fixture_node_sequence(fx, mode):
    """Same pop order, same per-node outcomes, same final tableau as the reference's loop --
    whatever the speculation width or evaluation back-end."""
    import jslpsolver_b200 as J
    from oracle import ref_model
    if fx["file"] == "Monster_II.json" and mode not in ("hbm_seq", "auto_spec8", "hbm_slots3_steps5", "auto_spec8_logcap3"):
        pytest.skip("large MIP: covered by two modes")
    if fx["file"] == "Vendor Selection.json" and mode != "auto_spec32":
        pytest.skip("long MIP: covered by one mode")
    if "k2" in fx and mode not in GENERATED_MODES:
        pytest.skip("generated MIP: covered by one mode per back end")
    jm = strip_timeouts(fx["model"])
    max_nodes = fx.get("max_nodes", 0)
    osol = ref_model.solve_full(jm, fast_cycles=True, node_log=1 << 20, max_nodes=max_nodes)
    if osol.tableau is None:
        pytest.skip("decided by presolve")
    s = J.Solver()
    s.engine, s.max_spec_batch = BNB_MODES[mode][:2]
    if len(BNB_MODES[mode]) > 2:
        s.node_slots, s.slot_steps = BNB_MODES[mode][2:4]
    if len(BNB_MODES[mode]) > 4:
        s.options = dict(BNB_MODES[mode][4])
    gsol = solve_capped(s, jm, max_nodes)
    gt = gsol._tableau
    assert_node_log_parity(gt, osol.tableau, fx["file"])
    if "k2" in fx:
        assert_backend(gt, fx, mode)
    st = osol.state
    assert gt.branchAndCutIterations == st.bncIterations
    assert (gt.feasible, gt.bounded) == (bool(st.feasible), bool(st.bounded))
    assert same_bits(gt.evaluation, st.evaluation), (fx["file"], gt.evaluation, st.evaluation)
    assert same_bits(gt.matrix2d(), osol.tableau.matrix())
    assert np.array_equal(gt.varIndexByRow, osol.tableau.maps()[0])
    assert [(a, b, float(c)) for a, b, c in gt.bestCuts] == [(a, b, float(c)) for a, b, c in osol.tableau.best_cuts()]


# ------------------------------------------------------------------ timeout / keep_solutions (branch-and-cut.ts:61-63,76,143-153)
def _fixture(name):
    return [f for f in BUNDLE["fixtures"] if f["file"] == name][0]


def test_timeout_stops_the_loop_with_the_incumbent_so_far():
    """model.timeout is wall clock (Date.now() < terminalTime before every iteration): whatever prefix of the loop ran
    must be the reference's prefix, and the result keeps the reference's shape.  A generous timeout changes nothing."""
    import jslpsolver_b200 as J
    from oracle import ref_model
    jm = strip_timeouts(_fixture("LargeFarmMIP.json")["model"])
    osol = ref_model.solve_full(jm, fast_cycles=True, node_log=1 << 20)
    onl = osol.tableau.node_log()
    full = J.Solve(dict(jm, timeout=600000))
    assert full == ref_model.Solve(jm, fast_cycles=True)
    for tmo in (0.5, 2.0, 5.0):
        s = J.Solver()
        s.max_spec_batch = 4
        gsol = s.Solve(dict(jm, timeout=tmo), full=True)
        gt = gsol._tableau
        b = gt.lastBnbStatus
        gnl = gt.node_log()
        assert len(gnl) == b.iterations <= len(onl)
        assert np.array_equal(gnl[:, [0, 1, 2, 4, 5, 7]], onl[:len(gnl), [0, 1, 2, 4, 5, 7]])
        if b.iterations < len(onl):
            assert b.timed_out == 1
        res = s._simplified(gsol)
        assert list(res)[:3] == ["feasible", "result", "bounded"] or "feasible" in res
        incumbents = [r for r in gnl if r[4] == 1]
        if incumbents:  # the winner is re-solved: the tableau holds the best incumbent so far
            assert same_bits(gt.evaluation, incumbents[-1][3]) and res.get("isIntegral") is True
    assert b.timed_out in (0, 1)


def test_keep_solutions_stores_every_incumbent():
    """options.keep_solutions: model.solutions gets one {var: value, ..., result} per incumbent, in order."""
    import jslpsolver_b200 as J
    from oracle import ref_model
    for name in ("LargeFarmMIP.json", "Knapsack 1.json", "Monster_II.json"):
        jm = strip_timeouts(_fixture(name)["model"])
        jm["options"] = dict(jm.get("options") or {}, keep_solutions=True)
        osol = ref_model.solve_full(jm, fast_cycles=True, node_log=1 << 20)
        onl = osol.tableau.node_log()
        s = J.Solver()
        gsol = s.Solve(jm, full=True)
        m = s.lastSolvedModel
        incumbents = [r for r in onl if r[4] == 1 and r[0] > 1]
        assert len(m.solutions or []) == len(incumbents), name
        sign = 1.0 if m.isMinimization else -1.0
        for sol, r in zip(m.solutions, incumbents):
            assert same_bits(sol["result"], sign * r[3]) or sol["result"] == sign * r[3]
        if incumbents:
            last = dict(m.solutions[-1])
            assert last.pop("result") == gsol.evaluation
            final = {k: v for k, v in gsol.solutionSet.items()}
            assert last == final, name
        assert s._simplified(gsol) == ref_model.Solve(jm, fast_cycles=True)


# ------------------------------------------------------------------ useMIRCuts (cutting-strategies.ts:74-212, branch-and-cut.ts:38-51)
def test_mir_primitives_match_oracle():
    """addLowerBoundMIRCut / addUpperBoundMIRCut / applyMIRCuts / computeFractionalVolume on a solved root, bit for bit."""
    from jslpsolver_b200 import problems
    it = problems.dense_packing_lp_tableau(19, 13, seed=4)
    it.integerIndices = np.array([13 + j for j in range(0, 19, 2)], dtype=np.int32)
    o = oracle_lp(it)
    g = gpu_lp(it, 2)
    o.simplex(); g.simplex()
    assert same_bits(g.computeFractionalVolume(True), o.fractional_volume(True))
    assert same_bits(g.computeFractionalVolume(False), o.fractional_volume(False))
    for r in range(0, o.state().height):
        assert g.addLowerBoundMIRCut(r) == o.add_mir_cut(r), r
    assert g.height == o.state().height and same_bits(g.matrix2d(), o.matrix())
    assert np.array_equal(g.varIndexByRow, o.maps()[0])
    for r in (1, 2, 5):
        assert g.addUpperBoundMIRCut(r) == o.add_mir_cut(r, upper=True), r
    assert same_bits(g.matrix2d(), o.matrix())
    o.simplex(); g.simplex()
    assert_lp_parity(g, o, "after MIR cuts")
    o.apply_mir_cuts(); g.applyMIRCuts()
    assert g.height == o.state().height and same_bits(g.matrix2d(), o.matrix())


@pytest.mark.parametrize("fx", MIP_FIXTURES + GENERATED_MIPS, ids=lambda f: f["file"])
def test_mip_fixture_with_mir_cuts_matches_oracle(fx):
    """options.useMIRCuts: same node sequence, same final tableau as the oracle's restatement of the MIR loop."""
    import jslpsolver_b200 as J
    from oracle import ref_model
    jm = strip_timeouts(fx["model"])
    jm["options"] = dict(jm.get("options") or {}, useMIRCuts=True)
    max_nodes = fx.get("max_nodes", 0)
    osol = ref_model.solve_full(jm, fast_cycles=True, node_log=1 << 20, max_nodes=max_nodes)
    if osol.tableau is None:
        pytest.skip("decided by presolve")
    s = J.Solver()
    s.max_spec_batch = 8
    gsol = solve_capped(s, jm, max_nodes)
    gt = gsol._tableau
    assert_node_log_parity(gt, osol.tableau, fx["file"])
    if "k2" in fx:   # the MIR loop runs on the single-tableau path: neither the node kernel nor node slots
        b = gt.lastBnbStatus
        assert b.node_kernel_ms == 0 and b.slot_pivots == 0, (b.node_kernel_ms, b.slot_pivots)
    assert gt.branchAndCutIterations == osol.state.bncIterations
    assert same_bits(gt.matrix2d(), osol.tableau.matrix())
    assert np.array_equal(gt.varIndexByRow, osol.tableau.maps()[0])
    assert s._simplified(gsol) == ref_model.simplify(osol)
    assert same_bits(gt.bestPossibleEval, osol.state.bestPossibleEval) and gt.lastBnbStatus.feasible == osol.state.feasible


# ------------------------------------------------------------------ dynamic modification (dynamic-modification.ts:16-316)
def _same_state(g, o, what):
    assert g.height == o.state().height and g.width == o.state().width, what
    assert np.array_equal(g.varIndexByRow, o.maps()[0]) and np.array_equal(g.varIndexByCol, o.maps()[1]), what
    assert same_bits(g.matrix2d(), o.matrix()), f"{what}: tableau bits differ"


@pytest.mark.parametrize("seed", [31, 32, 33])
def test_dynamic_modification_sequence_matches_oracle(seed):
    """Edits on the device-resident tableau (right-hand sides, costs, coefficients, rows and columns added and removed),
    each followed by a re-solve, against the oracle's restatement of dynamic-modification.ts -- bit for bit."""
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    from oracle import ref_model
    rng = np.random.default_rng(seed)
    it = Model().loadJson(problems.mixed_lp_model(14, 10, seed)).initial_tableau()
    o = oracle_lp(it)
    g = gpu_lp(it, 2)
    o.simplex(); g.simplex()
    assert_lp_parity(g, o, "initial solve")
    H0, W0 = it.matrix.shape
    n_idx = H0 + W0 - 2

    def resolve(what):
        o.simplex(); g.simplex()
        _same_state(g, o, what + " / re-solve")
        st, os_ = g.lastStatus, o.state()
        assert (bool(st.feasible), bool(st.bounded)) == (bool(os_.feasible), bool(os_.bounded)), what
        if st.feasible and st.bounded:
            assert same_bits(st.evaluation, os_.evaluation), what

    vrow, vcol = o.maps()
    basic_slack = next(int(v) for v in vrow[1:] if v < H0 - 1)
    nonbasic = [int(v) for v in vcol[1:]]
    # updateRightHandSide: a constraint whose slack is basic, one whose slack is non-basic (if any)
    o.update_rhs(basic_slack, 2.5); g.updateRightHandSide(basic_slack, 2.5)
    _same_state(g, o, "updateRightHandSide (basic)")
    nb_slack = next((v for v in nonbasic if v < H0 - 1), None)
    if nb_slack is not None:
        o.update_rhs(nb_slack, -1.25); g.updateRightHandSide(nb_slack, -1.25)
        _same_state(g, o, "updateRightHandSide (non-basic)")
    resolve("updateRightHandSide")
    # updateCost: a basic and a non-basic structural variable
    vrow, vcol = o.maps()
    for v in ([int(x) for x in vrow[1:] if x >= H0 - 1][:1] + [int(x) for x in vcol[1:] if x >= H0 - 1][:1]):
        d = float(rng.integers(-5, 6)) + 0.5
        o.update_cost(v, d); g.updateCost(v, d)
        _same_state(g, o, f"updateCost {v}")
    resolve("updateCost")
    # updateConstraintCoefficient: may pivot the constraint's slack into the basis first (putInBase)
    vrow, vcol = o.maps()
    ci = int([v for v in list(vcol[1:]) + list(vrow[1:]) if v < H0 - 1][0])
    for vi in ([int(x) for x in vcol[1:] if x >= H0 - 1][:1] + [int(x) for x in vrow[1:] if x >= H0 - 1][:1]):
        o.update_coefficient(ci, vi, 1.75); g.updateConstraintCoefficient(ci, vi, 1.75)
        _same_state(g, o, f"updateConstraintCoefficient {ci},{vi}")
    with pytest.raises(ValueError):
        g.updateConstraintCoefficient(ci, ci, 1.0)
    resolve("updateConstraintCoefficient")
    # addConstraint with terms on basic and non-basic variables (rows grow past the initial capacity on the way)
    for k in range(3):
        vrow, vcol = o.maps()
        terms = [(int(vrow[1 + k]), 2.0 + k), (int(vcol[1 + k]), -1.5), (int(vcol[2 + k]), 0.75)]
        new_index = n_idx + k
        o.add_constraint(k % 2 == 0, 40.0 + k, new_index, terms)
        g.addConstraint(isUpperBound=k % 2 == 0, rhs=40.0 + k, index=new_index, terms=terms)
        _same_state(g, o, f"addConstraint {k}")
    resolve("addConstraint")
    # addVariable + coefficients on it
    new_var = n_idx + 3
    o.add_variable(new_var, -7.0); g.addVariable(index=new_var, cost=7.0)   # minimisation: entry = -cost
    _same_state(g, o, "addVariable")
    o.update_coefficient(ci, new_var, -2.0); g.updateConstraintCoefficient(ci, new_var, -2.0)
    _same_state(g, o, "coefficient on the new variable")
    resolve("addVariable")
    # putInBase / takeOutOfBase
    vrow, vcol = o.maps()
    v_nb, v_b = int(vcol[1]), int(vrow[2])
    assert g.putInBase(v_nb) == o.put_in_base(v_nb)
    _same_state(g, o, "putInBase")
    assert g.takeOutOfBase(v_b) == o.take_out_of_base(v_b)
    _same_state(g, o, "takeOutOfBase")
    # removeConstraint: swap with the last row.  (The reference leaves rowByVarIndex of the moved row stale,
    # dynamic-modification.ts:241-243; the oracle is rebuilt from its own tableau before going on.)
    slack = n_idx + 1
    o.remove_constraint(slack); g.removeConstraint(slack)
    _same_state(g, o, "removeConstraint")
    o2 = ref_model.OracleTableau(o.matrix(), *o.maps(), fast_cycles=True)
    o2.simplex(); g.simplex()
    _same_state(g, o2, "removeConstraint / re-solve")
    # removeVariable: the reference only decrements `width` and keeps indexing the un-compacted array; the device keeps
    # its row stride.  Compared on the reference's backing array viewed with the OLD width.
    vrow, vcol = o2.maps()
    H, W = o2.state().height, o2.state().width
    victim = int(vcol[2])
    o2.remove_variable(victim); g.removeVariable(victim)
    flat = o2.flat(H * W).reshape(H, W)[:, :W - 1]
    assert g.width == W - 1 and same_bits(g.matrix2d(), flat)
    assert np.array_equal(g.varIndexByCol, o2.maps()[1])
    o3 = ref_model.OracleTableau(flat.copy(), o2.maps()[0], o2.maps()[1], fast_cycles=True)
    o3.simplex(); g.simplex()
    _same_state(g, o3, "removeVariable / re-solve")


def test_model_level_edits_after_solve():
    """model.ts:196-273 through the host mirror: edit a solved model, solve again, compare with solving the edited model
    from scratch (same optimum; the pivot path differs, so values are compared to 1e-9 relative).  The bit-for-bit
    comparison of the same kind of edits with the oracle is test_gpu_dynamic_edges.test_model_edits_replayed_on_the_oracle."""
    import jslpsolver_b200 as J
    m = J.Model().loadJson({"optimize": "profit", "opType": "max",
                            "constraints": {"wood": {"max": 300}, "labor": {"max": 110}, "storage": {"max": 400}},
                            "variables": {"table": {"wood": 30, "labor": 5, "profit": 1200, "storage": 30},
                                          "dresser": {"wood": 20, "labor": 10, "profit": 1600, "storage": 50}}})
    s1 = m.solve()
    # optimum at wood and storage binding: table = 70/9, dresser = 10/3, profit = 44000/3
    assert s1.feasible and abs(s1.evaluation - 44000 / 3) <= 1e-9 * 44000 / 3, s1.evaluation
    wood = m.constraints[0]
    wood.setRightHandSide(360)                        # updateRightHandSide
    table = m.variables[0]
    m.setCost(1500, table)                            # updateCost
    chair = m.addVariable(700, "chair")               # addVariable + coefficients
    for c, a in zip(m.constraints, (10, 4, 12)):
        c.addTerm(a, chair)
    extra = m.smallerThan(25)                         # addConstraint: table + dresser + chair <= 25
    for v in m.variables:
        extra.addTerm(1, v)
    s2 = m.solve()
    fresh = J.Model().loadJson({"optimize": "profit", "opType": "max",
                                "constraints": {"wood": {"max": 360}, "labor": {"max": 110}, "storage": {"max": 400}, "count": {"max": 25}},
                                "variables": {"table": {"wood": 30, "labor": 5, "profit": 1500, "storage": 30, "count": 1},
                                              "dresser": {"wood": 20, "labor": 10, "profit": 1600, "storage": 50, "count": 1},
                                              "chair": {"wood": 10, "labor": 4, "profit": 700, "storage": 12, "count": 1}}})
    s3 = fresh.solve()
    assert s2.feasible and s3.feasible and abs(s2.evaluation - s3.evaluation) <= 1e-9 * abs(s3.evaluation)
    m.removeConstraint(extra)                         # removeConstraint
    s4 = m.solve()
    assert s4.feasible and s4.evaluation >= s2.evaluation - 1e-6


# ------------------------------------------------------------------ enhanced service (enhanced-branch-and-cut.ts)
ENHANCED = [{"nodeSelection": "hybrid"}, {"nodeSelection": "depth-first", "branching": "strong"},
            {"nodeSelection": "best-first", "branching": "most-fractional"}, {"branching": "pseudocost", "useMIRCuts": True},
            # options.useIncremental: the incremental service (parent checkpoints, incremental-branch-and-cut.ts)
            {"useIncremental": True}, {"useIncremental": True, "nodeSelection": "depth-first", "branching": "most-fractional"},
            {"useIncremental": True, "useMIRCuts": True}]


@pytest.mark.parametrize("opts", ENHANCED, ids=lambda o: "-".join(str(v) for v in o.values()))
@pytest.mark.parametrize("fx", MIP_FIXTURES + GENERATED_MIPS, ids=lambda f: f["file"])
def test_enhanced_service_matches_oracle(fx, opts):
    """options.nodeSelection / options.branching select the enhanced service (main.ts:62-83): same node sequence (stack /
    heap order, pseudocost-driven branching variables), same final tableau as the oracle's restatement."""
    import jslpsolver_b200 as J
    from oracle import ref_model
    if fx["file"] in ("Vendor Selection.json", "Monster_II.json") and "branching" in opts and opts.get("nodeSelection") != "depth-first":
        pytest.skip("long MIP: covered by two combinations")
    if "k2" in fx and opts != ENHANCED[0]:
        pytest.skip("generated MIP: covered by the hybrid / pseudocost service")
    jm = strip_timeouts(fx["model"])
    jm["options"] = dict(jm.get("options") or {}, **opts)
    max_nodes = fx.get("max_nodes", 0)
    osol = ref_model.solve_full(jm, fast_cycles=True, node_log=1 << 20, max_nodes=max_nodes)
    if osol.tableau is None:
        pytest.skip("decided by presolve")
    s = J.Solver()
    gsol = solve_capped(s, jm, max_nodes)
    gt = gsol._tableau
    assert_node_log_parity(gt, osol.tableau, fx["file"])
    assert gt.branchAndCutIterations == osol.state.bncIterations
    assert same_bits(gt.matrix2d(), osol.tableau.matrix())
    assert s._simplified(gsol) == ref_model.simplify(osol)


# ------------------------------------------------------------------ shape limits (DESIGN.md section 7)
def test_tall_tableau_takes_the_in_place_step_and_still_matches():
    """More than 32 rows per row CTA (H > ~9.4 k): the ping-pong step does not apply, the in-place step runs."""
    from jslpsolver_b200 import problems
    it = problems.dense_packing_lp_tableau(40, 10000, seed=8)
    o = oracle_lp(it)
    o.simplex()
    g = gpu_lp(it, 2)
    g.simplex()
    assert_lp_parity(g, o, "tall 10001 x 41")


def test_too_wide_tableau_fails_loudly():
    """The pivot row is staged whole in shared memory: beyond 25 600 columns jslp_tab_create reports JSLP_E_CAPACITY."""
    from jslpsolver_b200 import JslpError
    from jslpsolver_b200.tableau import GpuTableau
    M = np.zeros((3, 26001))
    g = GpuTableau(1e-8)
    with pytest.raises(JslpError, match="width exceeds"):
        g.upload(M, np.array([-1, 0, 1], dtype=np.int32), np.concatenate([[-1], 2 + np.arange(26000)]).astype(np.int32))


# ------------------------------------------------------------------ independent cross-check
def test_solve_agrees_with_an_independent_solver():
    """Solve() on the GPU against SciPy's HiGHS (no code or pivot rule shared with the reference or the oracle) on random
    LPs and small MIPs: same feasibility verdict, objective within 1e-7 relative."""
    pytest.importorskip("scipy")
    import jslpsolver_b200 as J
    from test_oracle_golden import _random_model, _scipy_solve
    rng = np.random.default_rng(77)
    checked = 0
    for k in range(40):
        model = _random_model(rng, int(rng.integers(3, 10)), int(rng.integers(2, 8)), k % 2 == 1)
        ok, val, status = _scipy_solve(model)
        if status not in (0, 2):
            continue
        res = J.Solve(model)
        assert bool(res["feasible"]) == ok, (k, res, status)
        if ok:
            assert res["bounded"] and abs(res["result"] - val) <= 1e-7 * max(1.0, abs(val)), (k, res["result"], val)
            checked += 1
    assert checked >= 20
    # mixed min / max / equal rows, both senses, either sign of cost: verdicts too (HiGHS status 0 / 2 / 3)
    from test_oracle_golden import _random_model_mixed, _scipy_solve_mixed
    rng = np.random.default_rng(6)
    seen = {0: 0, 2: 0, 3: 0}
    for k in range(90):
        model = _random_model_mixed(rng, int(rng.integers(3, 14)), int(rng.integers(2, 9)), k % 3 == 1)
        status, val = _scipy_solve_mixed(model)
        res = J.Solve(model)
        if status == 0:
            assert res["feasible"] and res["bounded"] and abs(res["result"] - val) <= 1e-7 * max(1.0, abs(val)), (k, res, val)
        elif status == 2:
            assert not res["feasible"], (k, res)
        elif status == 3:
            assert not (res["feasible"] and res["bounded"]), (k, res)
        seen[status] = seen.get(status, 0) + 1
    assert seen[0] >= 15 and seen[2] >= 15 and seen[3] >= 5, seen

"""The dynamic-modification API on the device (jslp_dynamic.cuh and the GpuTableau / Model methods that drive it) at
its launch-geometry, capacity and engine edges, bit for bit against the oracle.

Every edit kernel is a grid-stride loop of 256-thread CTAs: k_row_axpy over the width, k_col_axpy and k_copy_col over
the tableau rows and then the optional-objective rows, k_add_constraint and k_swap_rows over the row stride.  The cases
put each loop bound on 255 / 256 / 257 and 512 / 513, with the 256-row boundary once on a tableau row and once on an
optional-objective row.  addVariable at W == stride re-lays every buffer out at stride + 16 (restride), after solves on
each engine and after a ping-pong solve that left the tableau in the second buffer; addConstraint at H == rowcap grows
the rows by half plus 8, across the step grid's CTA count and across the L2 threshold of the step variant.  After every
edit and every re-solve the tableau bits, both label maps, the optional objectives and jslp_tab_info are compared; a
re-solve also compares status, evaluation bits and the pivots it made.

removeVariable: the reference only narrows `width` and reads its un-compacted array at the new width; the device keeps
its row stride (DESIGN.md section 7).  The oracle is compared on its backing array viewed at the old width and then
rebuilt from that view, as in test_gpu_lp_parity."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_lp_parity import (BNB_MODES, _same_state, assert_backend, assert_lp_parity, assert_node_log_parity,
                                oracle_lp, same_bits)

pytestmark = pytest.mark.gpu
LOG = 1 << 16


def ceil16(x):
    return (x + 15) // 16 * 16


def tab_info(g):
    """(W, H, nVars, lastElementIndex, stride, rowcap) as the device reports them."""
    from jslpsolver_b200 import _lib
    a = (C.c_int32 * 6)()
    _lib.check(g.context.lib.jslp_tab_info(g._h(), a))
    return tuple(a)


def upload(it, rowcap=None, engine=2):
    from jslpsolver_b200 import _lib
    from jslpsolver_b200.tableau import GpuTableau
    g = GpuTableau(1e-8)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, it.integerIndices, it.optionalCosts,
             row_capacity=rowcap)
    g.set_option(_lib.OPT_ENGINE, engine)
    g.set_option(_lib.OPT_PIVOT_LOG_CAP, LOG)
    g.optionalPriorities = list(getattr(it, "optionalPriorities", None) or range(1, g.nOpt + 1))
    return g


class Pair:
    """A device tableau and the oracle driven through the same edits, with the bookkeeping jslp_tab_info must show:
    lastElementIndex grows to cover every index an edit hands in, the stride by 16 when addVariable reaches it, the
    row capacity to max(H + 1, rowcap + rowcap / 2 + 8) when addConstraint reaches it."""

    def __init__(self, it, rowcap=None, engine=2, **okw):
        H, W = it.matrix.shape
        from oracle import ref_model
        self.it, self.g = it, upload(it, rowcap, engine)
        self.o = ref_model.OracleTableau(it.matrix, it.varIndexByRow, it.varIndexByCol, precision=1e-8,
                                         unrestricted=it.unrestricted, integers=it.integerIndices,
                                         opt_rc=it.optionalCosts, fast_cycles=True, pivot_log=LOG, **okw)
        self.okw = okw
        self.lei = H + W - 2
        self.n_vars = H + W - 2
        self.stride = ceil16(W)
        self.rowcap = rowcap if rowcap else H + 64
        self.unres = None if it.unrestricted is None else np.array(it.unrestricted, dtype=np.uint8)
        self.check("upload")

    @property
    def nOpt(self):
        return self.g.nOpt

    def check(self, what):
        g, o = self.g, self.o
        g._cache.clear()
        _same_state(g, o, what)
        if self.nOpt:
            assert same_bits(g.optional_reduced_costs(), o.optional()), f"{what}: optional objectives differ"
        s = o.state()
        assert tab_info(g) == (s.width, s.height, self.n_vars, self.lei, self.stride, self.rowcap), \
            (what, tab_info(g), (s.width, s.height, self.n_vars, self.lei, self.stride, self.rowcap))

    def resolve(self, what, engine=None):
        """Both sides re-solve; the pivots this solve made, flags, counts and evaluation bits must agree."""
        g, o = self.g, self.o
        n_g, n_o = len(g.pivot_log()), len(o.pivot_log())
        o.simplex()
        g.simplex()
        st, os_ = g.lastStatus, o.state()
        glog, olog = g.pivot_log()[n_g:], o.pivot_log()[n_o:]
        assert np.array_equal(glog, olog), f"{what}: pivots differ ({len(glog)} vs {len(olog)})"
        assert (bool(st.feasible), bool(st.bounded)) == (bool(os_.feasible), bool(os_.bounded)), what
        assert (st.phase1_pivots, st.phase2_pivots) == (os_.lastP1, os_.lastP2), what
        if st.feasible and st.bounded:
            assert same_bits(st.evaluation, os_.evaluation), what
        if engine is not None:
            assert (st.engine == 4) == (engine == 4), (what, st.engine)
        self.check(what + " / re-solve")
        return st

    # ---- edits, on both sides
    def update_rhs(self, ci, d):
        self.o.update_rhs(ci, d); self.g.updateRightHandSide(ci, d)
        self.check(f"updateRightHandSide {ci}")

    def update_coefficient(self, ci, vi, d):
        self.o.update_coefficient(ci, vi, d); self.g.updateConstraintCoefficient(ci, vi, d)
        self.check(f"updateConstraintCoefficient {ci},{vi}")

    def update_cost(self, vi, d, slot=-1):
        self.o.update_cost(vi, d, slot); self.g.updateCost(vi, d, priority=0 if slot < 0 else self.g.optionalPriorities[slot])
        self.check(f"updateCost {vi} slot {slot}")

    def add_constraint(self, up, rhs, idx, terms):
        H = self.o.state().height
        if H + 1 > self.rowcap:
            self.rowcap = max(H + 1, self.rowcap + self.rowcap // 2 + 8)
        self.o.add_constraint(up, rhs, idx, terms)
        self.g.addConstraint(isUpperBound=up, rhs=rhs, index=idx, terms=terms)
        self.lei = max(self.lei, idx + 1)
        self.check(f"addConstraint {idx} ({len(terms)} terms)")

    def remove_constraint(self, idx):
        assert self.o.remove_constraint(idx) == 0
        self.g.removeConstraint(idx)
        self.check(f"removeConstraint {idx}")
        self.rebuild(self.o.matrix())   # the reference leaves rowByVarIndex of the moved row stale

    def add_variable(self, vi, cost, slot=-1, is_integer=False, is_unrestricted=False):
        W = self.o.state().width
        if W + 1 > self.stride:
            self.stride += 16
        model = self.g.model
        entry = cost if model is not None and not model.isMinimization else -cost   # dynamic-modification.ts:252
        self.o.add_variable(vi, entry, slot, is_integer, is_unrestricted)
        self.g.addVariable(index=vi, cost=cost, priority=0 if slot < 0 else self.g.optionalPriorities[slot],
                           isInteger=is_integer, isUnrestricted=is_unrestricted)
        self.lei = max(self.lei, vi + 1)
        if is_unrestricted:
            u = np.zeros(max(len(self.unres), vi + 1), dtype=np.uint8)
            u[:len(self.unres)] = self.unres
            u[vi] = 1
            self.unres = u
        self.check(f"addVariable {vi}")

    def remove_variable(self, vi):
        s = self.o.state()
        H, W = s.height, s.width
        assert self.o.remove_variable(vi) == 0
        self.g.removeVariable(vi)
        self.g._cache.clear()
        flat = self.o.flat(H * W).reshape(H, W)[:, :W - 1]
        assert self.g.width == W - 1 and same_bits(self.g.matrix2d(), flat), f"removeVariable {vi}: tableau bits differ"
        assert np.array_equal(self.g.varIndexByCol, self.o.maps()[1]), f"removeVariable {vi}"
        if self.nOpt:
            assert same_bits(self.g.optional_reduced_costs(), self.o.optional()), f"removeVariable {vi}: optional"
        self.rebuild(flat.copy())
        self.check(f"removeVariable {vi}")

    def rebuild(self, M):
        from oracle import ref_model
        o = self.o
        vr, vc = o.maps()
        self.o = ref_model.OracleTableau(M, vr, vc, precision=1e-8, unrestricted=self.unres, integers=self.it.integerIndices,
                                         opt_rc=o.optional() if self.nOpt else None, fast_cycles=True, pivot_log=LOG,
                                         **self.okw)

    # ---- labels
    def basic(self, structural=None):
        vr = self.o.maps()[0]
        return [int(v) for v in vr[1:] if structural is None or (v >= self.n_cons) == structural]

    def nonbasic(self, structural=None):
        vc = self.o.maps()[1]
        return [int(v) for v in vc[1:] if structural is None or (v >= self.n_cons) == structural]


def packing(n_vars, n_cons, seed, n_opt=0, rowcap=None, engine=2, solve=True):
    """A dense packing LP (constraints 0..n_cons-1, variables after), optionally with n_opt seeded optional objectives
    of non-dyadic entries, solved on both sides."""
    from jslpsolver_b200 import problems
    it = problems.dense_packing_lp_tableau(n_vars, n_cons, seed)
    rng = np.random.default_rng(seed)
    it.optionalCosts = np.round(rng.uniform(-3, 3, (n_opt, n_vars + 1)), 2) / 7.0 if n_opt else np.zeros((0, n_vars + 1))
    it.optionalPriorities = list(range(1, n_opt + 1))
    p = Pair(it, rowcap, engine)
    p.n_cons = n_cons
    if solve:
        p.resolve("initial solve")
    return p


COEFS = (1 / 3, 0.1, 1e-17, -0.0)


# ------------------------------------------------------------------ k_row_axpy: the width
@pytest.mark.parametrize("target", ["row0", "opt"])
@pytest.mark.parametrize("W", [2, 255, 256, 257, 512, 513, 1025])
def test_row_axpy_across_the_width(W, target):
    """updateCost of a basic variable adds its row to the cost row or to an optional-objective row;
    updateConstraintCoefficient of a basic variable adds its row to the constraint's row."""
    p = packing(W - 1, 6, seed=W, n_opt=1 if target == "opt" else 0)
    slot = 0 if target == "opt" else -1
    basic = p.basic(structural=True)
    assert basic, "no basic structural variable"
    p.update_cost(basic[0], 1 / 3, slot)
    p.update_cost(basic[-1], -0.1, slot)
    p.update_coefficient(p.basic(structural=False)[0] if p.basic(structural=False) else p.nonbasic(False)[0], basic[0], 0.1)
    p.resolve("row axpy")


# ------------------------------------------------------------------ k_col_axpy / k_copy_col: tableau rows + optional rows
@pytest.mark.parametrize("n_opt", [0, 1, 2])
@pytest.mark.parametrize("rows", [255, 256, 257, 512, 513])
def test_column_edits_across_tableau_and_optional_rows(rows, n_opt):
    """H + nOpt = rows: updateRightHandSide of a non-basic slack (k_col_axpy over every row and optional row),
    addVariable (k_copy_col zeroing a column), removeVariable of column 1 and of the last column (k_copy_col)."""
    H = rows - n_opt
    p = packing(8, H - 1, seed=rows + n_opt, n_opt=n_opt)
    slacks = p.nonbasic(structural=False)
    assert slacks, "no non-basic slack"
    p.update_rhs(slacks[0], 1 / 3)
    p.update_rhs(p.basic(structural=False)[0], -0.1)
    n = p.lei
    p.add_variable(n, 0.1, slot=n_opt - 1)
    p.update_coefficient(p.basic(structural=False)[1], n, 1 / 3)
    p.resolve("col axpy")
    vc = p.o.maps()[1]
    p.remove_variable(int(vc[1]))
    p.remove_variable(int(p.o.maps()[1][-1]))
    p.resolve("remove variable")


# ------------------------------------------------------------------ k_add_constraint / k_swap_rows: the stride
@pytest.mark.parametrize("stride", [16, 256, 272, 512, 528])
def test_add_and_remove_constraint_across_the_stride(stride):
    p = packing(stride - 1, 12, seed=stride, solve=False)
    assert tab_info(p.g)[4] == stride
    p.remove_constraint(int(p.o.maps()[0][1]))        # unsolved: row 1 holds slack 0, swapped with the last row
    p.resolve("initial solve")
    vr, vc = p.o.maps()
    b = [int(v) for v in vr[1:]]
    nb = [int(v) for v in vc[1:]]
    nxt = 12 + stride - 1
    p.add_constraint(True, 10 / 3, nxt, [])
    p.add_constraint(False, 0.1, nxt + 1, [(nb[0], 1 / 3)])
    # basic and non-basic terms, one variable twice, non-dyadic coefficients (an FMA would change the bits)
    terms = [(b[k % len(b)] if k % 3 else nb[k % len(nb)], COEFS[k % 4] * (1 + k % 5)) for k in range(307)]
    terms += [(b[0], 0.1), (b[0], -1 / 3)]
    p.add_constraint(True, 7.0, nxt + 2, terms)
    p.add_constraint(False, -0.1, nxt + 3, terms[:40])
    p.remove_constraint(nxt + 3)                      # basic in the last row: the swapped row is the last row
    p.resolve("add constraint")
    p.remove_constraint(nxt + 1)
    p.resolve("remove constraint")


# ------------------------------------------------------------------ restride
def _pp_case(W, seed):
    """A packing LP solved on the ping-pong step with an odd number of pivots, so that the result is in the second
    buffer when addVariable re-lays both out."""
    for s in range(seed, seed + 8):
        p = packing(W - 1, 40, seed=s, solve=False)
        st = p.resolve("ping-pong solve")
        if (st.phase1_pivots + st.phase2_pivots) % 2 == 1:
            return p
    raise AssertionError("no odd pivot count among the seeds")


# the ping-pong step runs without optional objectives: its case has none
@pytest.mark.parametrize("engine,n_opt", [(e, k) for e in (0, 1, 2, 4) for k in (0, 2)] + [("pingpong", 0)])
@pytest.mark.parametrize("W", [16, 256, 512])
def test_add_variable_at_the_stride(W, engine, n_opt):
    if engine == "pingpong":
        p = _pp_case(W, seed=W)
    else:
        p = packing(W - 1, 10, seed=W + 3, n_opt=n_opt, engine=engine)
    W0, stride0 = p.o.state().width, p.stride
    assert W0 == stride0 == W
    p.g.save()
    before = p.g.matrix2d().copy()
    n = p.lei
    p.add_variable(n, 2 / 3, slot=n_opt - 1)
    assert tab_info(p.g)[4] == W + 16
    # a snapshot of the old layout is void: restore() leaves the widened tableau as it is
    p.g.restore()
    p.check("restore after restride")
    assert p.g.matrix2d().shape == (before.shape[0], W + 1)
    for r in p.basic(structural=False)[:3]:
        p.update_coefficient(r, n, -1 / 3)
    p.resolve("after restride", engine=None)
    # a second column, past the new width, then a re-solve and the analyses that size buffers from the stride
    p.add_variable(n + 1, 0.1, slot=-1)
    p.update_coefficient(p.basic(structural=False)[0], n + 1, 0.5)
    p.resolve("second column")
    if not n_opt:
        _sensitivity_and_parametric(p)
    # removeVariable then addVariable: the freed column is reused, the stride stays
    p.remove_variable(int(p.o.maps()[1][1]))
    p.add_variable(n + 2, 1 / 3, slot=-1)
    assert tab_info(p.g)[4] == W + 16
    p.resolve("reuse")


def _sensitivity_and_parametric(p):
    from oracle import parametric as OP, sensitivity as S
    g, o = p.g, p.o
    if not (g.feasible and g.bounded):
        return
    unres = p.unres
    want = S.bounds(o.matrix(), *o.maps(), unres, 1e-8)
    got = g.sensitivity_bounds()
    assert all(same_bits(a, b) for a, b in zip(got, want)), "sensitivity bounds differ"
    M, (vr, vc) = o.matrix(), o.maps()
    lab = (p.nonbasic(False) or p.basic(False))[0]
    w = OP.path(M, vr, vc, unres, 1e-8, 0, [lab], [1.0], 0.0, 50.0, 16)
    a = g.parametric_path(0, [lab], [1.0], 0.0, 50.0, 16)
    n = len(w["records"])
    assert a["stop"] == w["stop"] and len(a["theta"]) == n
    ww = np.array([x[:3] for x in w["records"]], dtype=np.float64).reshape(n, 3)
    assert same_bits(np.stack([a["theta"], a["obj_raw"], a["dobj"]], axis=1).reshape(n, 3), ww)


# ------------------------------------------------------------------ row growth
def test_add_constraint_from_full_capacity_across_the_step_grid():
    """H == rowcap, then one addConstraint at a time: the capacity grows to rowcap + rowcap / 2 + 8 and takes the step
    grid (min(num_sms * 2, rowcap) CTAs) past num_sms * 2."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cap = 2 * sms - 6
    p = packing(20, cap - 1, seed=5, rowcap=cap)
    assert tab_info(p.g)[1] == tab_info(p.g)[5] == cap
    nb = p.nonbasic()
    for k in range(4):
        p.add_constraint(k % 2 == 0, 1 + k / 3, p.lei, [(nb[k], 0.1), (p.basic(True)[0], 1 / 3)])
    assert tab_info(p.g)[5] == cap + cap // 2 + 8 > 2 * sms
    p.resolve("grid change")
    for k in range(2):
        p.remove_constraint(int(p.o.maps()[0][-1]))
    p.resolve("after removals")


def test_row_growth_across_the_l2_threshold_of_the_step_variant():
    """16 * rowcap * stride crosses 0.95 * L2 through grow_rows: the step flips to the deeper-prefetch variant.  The
    tableau is feasible and one pivot from optimal, so the re-solves take a handful of pivots."""
    import torch
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    W = 1750
    stride = ceil16(W)
    H = int(0.95 * l2 / (16 * stride))        # the last row count below the threshold
    assert 16 * H * stride <= 0.95 * l2 < 16 * (H + H // 2 + 8) * stride
    rng = np.random.default_rng(3)
    from jslpsolver_b200.model import InitialTableau
    M = np.round(rng.uniform(0.1, 1.0, (H, W)), 3)
    M[1:, 0] = np.round(rng.uniform(5, 10, H - 1), 2)
    M[0, :] = 0.0
    M[0, 1:4] = (-1 / 3, 0.1, 0.7)
    vrow = np.array([-1] + list(range(H - 1)), dtype=np.int32)
    vcol = np.array([-1] + list(range(H - 1, H + W - 2)), dtype=np.int32)
    it = InitialTableau(M, vrow, vcol, np.zeros(H + W - 2, dtype=np.uint8), np.zeros(0, dtype=np.int32), [],
                        np.zeros((0, W)))
    p = Pair(it, rowcap=H)
    p.n_cons = H - 1
    p.resolve("below the threshold")
    p.add_constraint(True, 3.0, p.lei, [(int(p.o.maps()[1][5]), 1 / 3), (int(p.o.maps()[1][9]), 0.1)])
    W_, H_, _, _, s_, cap_ = tab_info(p.g)
    assert 16 * cap_ * s_ > 0.95 * l2 and cap_ == H + H // 2 + 8
    p.resolve("above the threshold")


# ------------------------------------------------------------------ the resident engine's H * W <= 16384
def test_edits_across_the_resident_engine_boundary():
    p = packing(127, 127, seed=12, engine=0)          # 128 x 128 = 16384: resident
    assert p.g.lastStatus.engine == 4
    p.add_constraint(True, 50.0, p.lei, [(p.nonbasic()[0], 1 / 3), (p.basic(True)[0], 0.1)])
    p.resolve("129 x 128", engine=2)
    p.remove_constraint(int(p.o.maps()[0][-1]))
    p.resolve("128 x 128 again", engine=4)
    p.add_variable(p.lei, 0.7)
    p.update_coefficient(p.basic(False)[0], p.lei - 1, 1 / 3)
    p.resolve("128 x 129", engine=2)
    p.remove_variable(int(p.o.maps()[1][-1]))
    p.resolve("128 x 128 after removeVariable", engine=4)


# ------------------------------------------------------------------ optional objectives from soft constraints
def _soft_model(levels, seed):
    rng = np.random.default_rng(seed)
    cons, variables = {}, {f"x{j}": {"profit": float(rng.integers(1, 30))} for j in range(10)}
    for i in range(14):
        spec = {"max": float(rng.integers(20, 60))}
        if i % 3 == 1:
            spec["priority"] = 1 + (i // 3) % levels
            spec["weight"] = float(rng.integers(1, 4))
        cons[f"c{i}"] = spec
        for j in range(10):
            if rng.random() < 0.6:
                variables[f"x{j}"][f"c{i}"] = float(rng.integers(1, 9)) / 3
    return {"optimize": "profit", "opType": "max", "constraints": cons, "variables": variables}


@pytest.mark.parametrize("levels", [2, 3])
def test_optional_objectives_of_soft_constraints(levels):
    from jslpsolver_b200.model import Model
    m = Model().loadJson(_soft_model(levels, seed=levels))
    it = m.initial_tableau()
    assert len(it.optionalPriorities) == levels
    p = Pair(it)
    p.n_cons = len(m.constraints)
    p.resolve("initial solve")
    prio = {v.index: v.priority for v in m.variables}
    for k in range(levels):
        slot = k
        vars_k = [v for v, pr in prio.items() if pr == k + 1]
        for v in vars_k:
            if v in p.basic() or v in p.nonbasic():
                p.update_cost(v, 1 / 3 if v in p.basic() else -0.1, slot)
        p.update_cost(p.basic(True)[0], 0.1, slot)
        p.update_cost(p.nonbasic()[0], 1 / 3, slot)
    slack = next(v for v in p.nonbasic() if v < p.n_cons and prio.get(v) is None)
    p.update_rhs(slack, 0.1)
    p.resolve("cost and rhs edits")
    n = p.lei
    for k in range(levels):
        p.add_variable(n + k, 0.5 + k / 3, slot=k)
        p.update_coefficient(p.basic(False)[0], n + k, 1 / 3)
    p.resolve("addVariable at each priority")
    for v in (int(p.o.maps()[1][1]), int(p.o.maps()[1][-1])):
        p.remove_variable(v)
    p.resolve("removeVariable")


# ------------------------------------------------------------------ integer / unrestricted variables added after a solve
@pytest.mark.parametrize("mode", ["auto_spec8", "hbm_spec4", "hbm_seq"])
def test_integer_and_unrestricted_variables_added_after_a_solve(mode):
    """addVariable(isInteger / isUnrestricted) with indices past the uploaded index arrays, then branch and cut, node
    log and all, on the resident node kernel, node slots and the one-node HBM path."""
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    m = Model().loadJson(problems.half_tie_mip_model(80, seed=80))
    m.max_nodes = 120
    it = m.initial_tableau()
    engine, spec = BNB_MODES[mode][:2]
    p = Pair(it, engine=engine, is_min=m.isMinimization, max_nodes=120, node_log=1 << 20)
    p.n_cons = len(m.constraints)
    g = p.g
    g.model, g.max_spec_batch = m, spec
    if len(BNB_MODES[mode]) > 2:
        g.node_slots, g.slot_steps = BNB_MODES[mode][2:4]
    p.resolve("root")
    n = p.lei
    rows = p.basic(False)[:2]
    p.add_variable(n, -2.5, is_integer=True)         # maximisation: the column takes the cost as is
    p.update_coefficient(rows[0], n, -2.0)
    p.add_variable(n + 1, -0.5, is_unrestricted=True)
    p.update_coefficient(rows[1], n + 1, -1.0)
    p.add_variable(n + 7, -1.5, is_integer=True, is_unrestricted=True)
    p.update_coefficient(rows[0], n + 7, -1 / 3)
    p.o.branch_and_cut()
    g.branchAndCut()
    assert_node_log_parity(g, p.o, mode)
    assert_backend(g, {"file": "half_tie_80 + added columns", "k2": True}, mode)
    assert g.branchAndCutIterations == p.o.state().bncIterations
    assert same_bits(g.matrix2d(), p.o.matrix())
    assert np.array_equal(g.varIndexByRow, p.o.maps()[0])


# ------------------------------------------------------------------ model level, replayed on the oracle
def _replay(p, calls):
    for call in calls:
        name, args = call[0], call[1:]
        o = p.o
        if name == "remove_variable":
            s = o.state()
            H, W = s.height, s.width
            assert o.remove_variable(args[0]) == 0
            p.rebuild(o.flat(H * W).reshape(H, W)[:, :W - 1].copy())
        elif name == "remove_constraint":
            assert o.remove_constraint(args[0]) == 0
            p.rebuild(o.matrix())
        elif name == "add_variable":
            o.add_variable(args[0], args[1], args[2], args[3], args[4])
        elif name == "add_constraint":
            o.add_constraint(*args)
        elif name == "update_cost":
            o.update_cost(args[0], args[2], args[1])
        else:
            getattr(o, name)(*args)


def test_model_edits_replayed_on_the_oracle():
    """Model API edits after a solve (max, Equality, relaxed rows at two priorities, availableIndexes reuse): after
    each re-solve the device tableau equals the oracle driven through the index-level calls the CPU suite pins."""
    from jslpsolver_b200 import _lib
    from jslpsolver_b200.model import Model
    from test_dynamic_edges_cpu import EDIT_MODEL, edit_stages, record_edit_calls
    it, stages = record_edit_calls()
    m = Model().loadJson(EDIT_MODEL)
    m.usePresolve = False
    m.tableau.options = {_lib.OPT_PIVOT_LOG_CAP: LOG}
    m.solve()
    g = m.tableau
    p = Pair.__new__(Pair)
    p.it, p.g, p.okw = it, g, {}
    p.o = oracle_lp(it)
    p.unres = it.unrestricted
    p.o.simplex()
    assert_lp_parity(g, p.o, "model solve")
    for k, (stage, calls) in enumerate(zip(edit_stages(m), stages)):
        stage()
        _replay(p, calls)
        n_g, n_o = len(g.pivot_log()), len(p.o.pivot_log())
        sol = m.solve()
        p.o.simplex()
        g._cache.clear()
        _same_state(g, p.o, f"stage {k + 1}")
        assert np.array_equal(g.pivot_log()[n_g:], p.o.pivot_log()[n_o:]), f"stage {k + 1}: pivots differ"
        if p.o.nOpt:
            assert same_bits(g.optional_reduced_costs(), p.o.optional()), f"stage {k + 1}"
        st = p.o.state()
        assert (sol.feasible, sol.bounded) == (bool(st.feasible), bool(st.bounded))
        if st.feasible and st.bounded:
            assert same_bits(g.lastStatus.evaluation, st.evaluation), f"stage {k + 1}"


# ------------------------------------------------------------------ takeOutOfBase past the row
def test_take_out_of_base_refuses_a_column_past_the_row():
    """Height > width with the variable's row zero past its right-hand side: the reference's flat scan would stop on
    the next row's right-hand side (tests/test_dynamic_edges_cpu.py pins that); the device reports no pivot element
    and leaves the tableau as it was, as the oracle does."""
    from jslpsolver_b200 import JslpError
    from jslpsolver_b200.model import InitialTableau
    H, W = 8, 4
    M = np.zeros((H, W))
    M[:, 0] = 1.0
    M[2:, 1:] = 0.5
    M[3, 1:] = 0.0
    vrow = np.array([-1] + list(range(H - 1)), dtype=np.int32)
    vcol = np.array([-1] + list(range(H - 1, H + W - 2)), dtype=np.int32)
    it = InitialTableau(M, vrow, vcol, np.zeros(H + W - 2, dtype=np.uint8), np.zeros(0, dtype=np.int32), [],
                        np.zeros((0, W)))
    p = Pair(it)
    assert p.o.take_out_of_base(int(vrow[3])) == -2
    with pytest.raises(JslpError, match="no pivot element"):
        p.g.takeOutOfBase(int(vrow[3]))
    with pytest.raises(JslpError, match="no pivot element"):
        p.g.removeVariable(int(vrow[3]))
    p.check("refused takeOutOfBase")

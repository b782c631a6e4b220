"""The dynamic-modification API on the CPU: the oracle's orc_dm_* against a literal restatement of
dynamic-modification.ts, and the index-level calls the host Model mirror makes for each model-level edit.

TsTableau below keeps the reference's data layout: one flat Float64Array for the matrix (removeVariable only
narrows `width`, so the rows after it are read at the new width from the old layout) and one reducedCosts array per
optional objective (indexed by column alone, so removeVariable moves none of them).  The oracle keeps its optional
objectives in one nOpt x W block; these tests pin that it still sits where separate arrays would, bit for bit, with
0 to 3 objectives and the victim column first, in the middle and last.

The second half drives jslpsolver_b200.model.Model through a GpuTableau whose C library records its calls instead of
reaching a device: updateRightHandSide / setCost signs, Equality fanning out to both rows, availableIndexes reuse and
priority -> optional-objective slot.  tests/test_gpu_dynamic_edges.py replays the same sequence on the oracle."""
import ctypes as C

import numpy as np
import pytest

from oracle import ref_model


def same_bits(a, b):
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all(a.view(np.uint64) == b.view(np.uint64)))


def _small(v):  # !(v >= -1e-16 && v <= 1e-16)
    return v >= -1e-16 and v <= 1e-16


# ------------------------------------------------------------------ restatement of dynamic-modification.ts
class TsTableau:
    def __init__(self, M, vrow, vcol, opt=None, precision=1e-8):
        M = np.asarray(M, dtype=np.float64)
        self.height, self.width = M.shape
        self.matrix = [float(x) for x in M.ravel()]
        self.varIndexByRow = [int(v) for v in vrow]
        self.varIndexByCol = [int(v) for v in vcol]
        self.rowByVarIndex, self.colByVarIndex = {}, {}
        for r in range(1, self.height):
            self.rowByVarIndex[self.varIndexByRow[r]] = r
            self.colByVarIndex[self.varIndexByRow[r]] = -1
        for c in range(1, self.width):
            self.colByVarIndex[self.varIndexByCol[c]] = c
            self.rowByVarIndex[self.varIndexByCol[c]] = -1
        self.optional = [[float(x) for x in row] for row in (opt if opt is not None else [])]
        self.precision = precision

    # simplex.ts:330-413
    def pivot(self, pr, pc):
        m, W, H = self.matrix, self.width, self.height
        po = pr * W
        quotient = m[po + pc]
        leaving, entering = self.varIndexByRow[pr], self.varIndexByCol[pc]
        self.varIndexByRow[pr] = entering
        self.varIndexByCol[pc] = leaving
        self.rowByVarIndex[entering] = pr
        self.rowByVarIndex[leaving] = -1
        self.colByVarIndex[entering] = -1
        self.colByVarIndex[leaving] = pc
        nz = []
        for c in range(W):
            val = m[po + c]
            if not _small(val):
                m[po + c] = val / quotient
                nz.append(c)
            else:
                m[po + c] = 0.0
        m[po + pc] = 1 / quotient
        for r in range(H):
            if r == pr:
                continue
            ro = r * W
            coefficient = m[ro + pc]
            if not _small(coefficient):
                for c in nz:
                    v0 = m[po + c]
                    if not _small(v0):
                        m[ro + c] = m[ro + c] - coefficient * v0
                    elif v0 != 0:
                        m[po + c] = 0.0
                m[ro + pc] = -coefficient / quotient
        for rc in self.optional:
            coefficient = rc[pc]
            if coefficient != 0:
                for c in nz:
                    v0 = m[po + c]
                    if v0 != 0:
                        rc[c] = rc[c] - coefficient * v0
                rc[pc] = -coefficient / quotient

    # :16-34 (returns -2 where the reference would call pivot(-1, c)).  addVariable gives its index no
    # rowByVarIndex entry (undefined: the reference's putInBase would return it unpivoted); the oracle and the device
    # read -1 there, and so does this restatement.
    def put_in_base(self, v):
        W, r = self.width, self.rowByVarIndex.get(v, -1)
        if r == -1:
            c = self.colByVarIndex[v]
            for r1 in range(1, self.height):
                x = self.matrix[r1 * W + c]
                if x < -self.precision or self.precision < x:
                    r = r1
                    break
            if r == -1:
                return -2
            self.pivot(r, c)
        return r

    # :36-55: the scan runs to the HEIGHT over the flat array; returns the column it found even when it lies past
    # the row (the reference would then pivot on an entry of a following row) and then does not pivot
    def take_out_of_base(self, v):
        W, c = self.width, self.colByVarIndex[v]
        if c == -1:
            r = self.rowByVarIndex[v]
            for c1 in range(1, self.height):
                k = r * W + c1
                x = self.matrix[k] if k < len(self.matrix) else float("nan")   # undefined: both tests false
                if x < -self.precision or self.precision < x:
                    c = c1
                    break
            if c == -1 or c >= W:
                return -2 if c == -1 else c
            self.pivot(r, c)
        return c

    # :78-106
    def update_rhs(self, ci, d):
        m, W = self.matrix, self.width
        row = self.rowByVarIndex[ci]
        if row == -1:
            sc = self.colByVarIndex[ci]
            for r in range(self.height):
                m[r * W] -= d * m[r * W + sc]
            for rc in self.optional:
                rc[0] -= d * rc[sc]
        else:
            m[row * W] -= d

    # :108-135
    def update_coefficient(self, ci, vi, d):
        m, W = self.matrix, self.width
        r = self.put_in_base(ci)
        cv = self.colByVarIndex[vi]
        if cv == -1:
            rv = self.rowByVarIndex[vi]
            for c in range(W):
                m[r * W + c] += d * m[rv * W + c]
        else:
            m[r * W + cv] -= d

    # :137-160 (slot -1: priority 0)
    def update_cost(self, vi, d, slot=-1):
        m, W = self.matrix, self.width
        col = self.colByVarIndex[vi]
        if col == -1:
            ro = self.rowByVarIndex[vi] * W
            dst = None if slot < 0 else self.optional[slot]
            for c in range(W):
                if dst is None:
                    m[c] += d * m[ro + c]
                else:
                    dst[c] += d * m[ro + c]
        else:
            m[col] -= d

    # :162-217
    def add_constraint(self, is_upper, rhs, slack, terms):
        sign = 1 if is_upper else -1
        last, W = self.height, self.width
        need = (last + 1) * W
        if len(self.matrix) < need:
            self.matrix += [0.0] * max(W * 16, len(self.matrix) // 2)
        m = self.matrix
        off = last * W
        for c in range(W):
            m[off + c] = 0.0
        m[off] = sign * rhs
        for v, coef in terms:
            vr = self.rowByVarIndex[v]
            if vr == -1:
                m[off + self.colByVarIndex[v]] += sign * coef
            else:
                for c in range(W):
                    m[off + c] -= sign * coef * m[vr * W + c]
        if len(self.varIndexByRow) <= last:
            self.varIndexByRow.append(slack)
        self.varIndexByRow[last] = slack
        self.rowByVarIndex[slack] = last
        self.colByVarIndex[slack] = -1
        self.height += 1

    # :219-245
    def remove_constraint(self, slack):
        m, W, last = self.matrix, self.width, self.height - 1
        r = self.put_in_base(slack)
        if r < 0:
            return -2
        for c in range(W):
            m[last * W + c], m[r * W + c] = m[r * W + c], m[last * W + c]
        self.varIndexByRow[r] = self.varIndexByRow[last]
        self.varIndexByRow[last] = -1
        self.rowByVarIndex[slack] = -1
        self.height -= 1
        return 0

    # :247-293 (slot -1: priority 0)
    def add_variable(self, vi, cost_entry, slot=-1):
        old, new, H = self.width, self.width + 1, self.height
        nm = [0.0] * (H * new)
        for r in range(H):
            nm[r * new:r * new + old] = self.matrix[r * old:r * old + old]
        self.matrix, self.width = nm, new
        last = new - 1
        for rc in self.optional:
            if len(rc) <= last:
                rc += [0.0] * (last + 1 - len(rc))
            rc[last] = 0.0
        if slot < 0:
            nm[last] = cost_entry
        else:
            self.optional[slot][last] = cost_entry
            nm[last] = 0.0
        self.colByVarIndex[vi] = last
        if len(self.varIndexByCol) <= last:
            self.varIndexByCol.append(vi)
        self.varIndexByCol[last] = vi

    # :295-316
    def remove_variable(self, vi):
        m, W = self.matrix, self.width
        last = W - 1
        c = self.take_out_of_base(vi)
        if c < 0:
            return -2
        for r in range(self.height):
            m[r * W + c] = m[r * W + last]
        self.varIndexByCol[c] = self.varIndexByCol[last]
        self.rowByVarIndex[vi] = -1
        self.colByVarIndex[vi] = -1
        self.width -= 1
        return 0

    def flat(self):
        return np.array(self.matrix[:self.height * self.width])

    def opt(self):
        return np.array([rc[:self.width] for rc in self.optional]).reshape(len(self.optional), self.width)


# ------------------------------------------------------------------ seeded tableaux
def _tableau(seed, H, W, n_opt):
    """A random H x W tableau in the shape Tableau._resetMatrix leaves (slack labels on rows, structural labels on
    columns), with non-dyadic entries so every product rounds, and n_opt optional-objective rows."""
    rng = np.random.default_rng(seed)
    M = np.round(rng.uniform(-4, 4, (H, W)), 2) / 3.0
    M[1:, 0] = np.abs(M[1:, 0]) + 1.0
    M[rng.random((H, W)) < 0.2] = 0.0
    vrow = np.array([-1] + list(range(H - 1)), dtype=np.int32)
    vcol = np.array([-1] + list(range(H - 1, H + W - 2)), dtype=np.int32)
    opt = np.round(rng.uniform(-3, 3, (n_opt, W)), 2) / 7.0
    return M, vrow, vcol, opt


def _pair(seed, H, W, n_opt):
    M, vrow, vcol, opt = _tableau(seed, H, W, n_opt)
    o = ref_model.OracleTableau(M, vrow, vcol, opt_rc=opt if n_opt else None)
    t = TsTableau(M, vrow, vcol, opt)
    for r, c0 in ((1, 2), (3, 1), (2, W - 1)):   # a few pivots so basic and non-basic labels mix
        cur = o.matrix()
        c = next(c for c in list(range(c0, W)) + list(range(1, c0)) if abs(cur[r, c]) > 0.05)
        o.pivot(r, c)
        t.pivot(r, c)
    return o, t


def _same(o, t, what):
    s = o.state()
    assert (s.height, s.width) == (t.height, t.width), what
    assert same_bits(o.flat(s.height * s.width), t.flat()), f"{what}: matrix bits differ"
    vr, vc = o.maps()
    assert list(vr) == t.varIndexByRow[:t.height] and list(vc) == t.varIndexByCol[:t.width], what
    if t.optional:
        assert same_bits(o.optional(), t.opt()), f"{what}: optional objectives differ"


def _labels(t):
    basic = [v for v in t.varIndexByRow[1:t.height]]
    nonbasic = [v for v in t.varIndexByCol[1:t.width]]
    return basic, nonbasic


@pytest.mark.parametrize("n_opt", [0, 1, 2, 3])
def test_every_edit_matches_the_restatement(n_opt):
    o, t = _pair(100 + n_opt, 9, 8, n_opt)
    _same(o, t, "after pivots")
    basic, nonbasic = _labels(t)
    slot = n_opt - 1 if n_opt else -1
    steps = [
        ("update_rhs", basic[0], 0.1), ("update_rhs", nonbasic[0], -1 / 3),
        ("update_coefficient", basic[1], nonbasic[1], 0.1), ("update_coefficient", nonbasic[2], basic[2], -1 / 3),
        ("update_cost", basic[3], 0.1, -1), ("update_cost", nonbasic[3], 1e-17, -1),
        ("update_cost", basic[4], -1 / 3, slot), ("update_cost", nonbasic[4], 0.7, slot),
        ("add_constraint", True, 10 / 3, 40, [(basic[0], 1 / 3), (nonbasic[0], 0.1), (basic[0], -0.0), (nonbasic[5], 1e-17)]),
        ("add_constraint", False, 0.1, 41, []),
        ("add_variable", 42, -1 / 3, slot), ("add_variable", 43, 0.1, -1),
        ("update_coefficient", 41, 42, 0.3), ("put_in_base", 42), ("take_out_of_base", 40),
        ("remove_constraint", 41),
    ]
    for step in steps:
        name, args = step[0], step[1:]
        a, b = getattr(o, name)(*args), getattr(t, name)(*args)
        if name in ("put_in_base", "take_out_of_base", "remove_constraint"):
            assert a == b, step
        _same(o, t, str(step))


@pytest.mark.parametrize("n_opt", [0, 1, 2, 3])
@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_remove_variable_keeps_each_optional_objective_in_place(n_opt, where):
    """removeVariable narrows the width; the oracle's optional objectives must stay where the reference's per-objective
    arrays leave them, through a later addVariable and right-hand-side / cost edits on an optional slot."""
    o, t = _pair(200 + n_opt, 8, 9, n_opt)
    _, nonbasic = _labels(t)
    col = {"first": 1, "middle": t.width // 2, "last": t.width - 1}[where]
    victim = t.varIndexByCol[col]
    assert o.remove_variable(victim) == t.remove_variable(victim) == 0
    _same(o, t, "removeVariable")
    slot = n_opt - 1 if n_opt else -1
    o.add_variable(50, 2 / 3, slot); t.add_variable(50, 2 / 3, slot)
    _same(o, t, "addVariable")
    basic, nonbasic = _labels(t)
    slack_nb = next(v for v in nonbasic if v < 7)
    for name, args in (("update_rhs", (slack_nb, 0.1)), ("update_rhs", (basic[0], 1 / 3)),
                       ("update_cost", (basic[1], 0.1, slot)), ("update_cost", (50, 1 / 3, slot)),
                       ("update_cost", (basic[2], -0.3, 0 if n_opt else -1))):
        getattr(o, name)(*args); getattr(t, name)(*args)
        _same(o, t, f"{name}{args}")


def test_remove_variable_scrambles_the_matrix_like_the_reference():
    """The matrix stays in the old layout read at the new width (the device keeps its row stride instead: DESIGN.md
    section 7); pinned so that a change to either side is a decision, not an accident."""
    o, t = _pair(7, 6, 6, 0)
    victim = t.varIndexByCol[2]
    expect = o.matrix()
    expect[:, 2] = expect[:, 5]                 # the last column copied over the victim's, rows left at width 6
    o.remove_variable(victim); t.remove_variable(victim)
    _same(o, t, "removeVariable")
    assert same_bits(o.flat(6 * 5), expect.ravel()[:30])
    assert same_bits(o.matrix()[1], expect.ravel()[5:10])   # row 1 at width 5 begins with old row 0's last entry


def test_take_out_of_base_scan_runs_past_the_row_when_height_exceeds_width():
    """takeOutOfBase scans columns 1 .. height-1 of the flat matrix.  With the variable's row zero past its right-hand
    side and height > width, the reference's scan reaches into the next row and stops at "column" width, the next
    row's right-hand side (it would then pivot on an entry outside the row); the oracle reports no pivot and leaves the
    tableau alone.  With height < width, a non-zero past column height-1 is never seen."""
    H, W = 8, 4
    M = np.zeros((H, W))
    M[:, 0] = 1.0
    M[2:, 1:] = 0.5
    M[3, 1:] = 0.0          # row 3: the victim's row, zero in every column
    vrow = np.array([-1] + list(range(H - 1)), dtype=np.int32)
    vcol = np.array([-1] + list(range(H - 1, H + W - 2)), dtype=np.int32)
    o = ref_model.OracleTableau(M, vrow, vcol)
    t = TsTableau(M, vrow, vcol)
    victim = int(vrow[3])
    assert t.take_out_of_base(victim) == W
    assert o.take_out_of_base(victim) == -2
    assert o.remove_variable(victim) == -2
    assert same_bits(o.matrix(), M) and list(o.maps()[0]) == list(vrow)
    # height < width: the row's only non-zero lies in column W-1 >= height, out of the scan
    M2 = np.zeros((3, 6)); M2[:, 0] = 1.0; M2[1, 5] = 2.0
    vr2, vc2 = np.array([-1, 0, 1], dtype=np.int32), np.array([-1, 2, 3, 4, 5, 6], dtype=np.int32)
    o2, t2 = ref_model.OracleTableau(M2, vr2, vc2), TsTableau(M2, vr2, vc2)
    assert t2.take_out_of_base(0) == o2.take_out_of_base(0) == -2


def test_add_variable_flags_extend_the_integer_and_unrestricted_sets():
    """orc_dm_add_variable(is_integer, is_unrestricted): the new index goes to the end of integerVariables
    (model.ts:169-176), so the MIP scan sees it; the default adds a continuous column.  max x + y, x <= 10, 2y <= 3."""
    M = np.array([[0.0, 1.0], [10.0, 1.0], [3.0, 0.0]])
    vrow, vcol = np.array([-1, 0, 1], dtype=np.int32), np.array([-1, 2], dtype=np.int32)
    picks = []
    for flags in ({}, {"is_integer": True}, {"is_integer": True, "is_unrestricted": True}):
        o = ref_model.OracleTableau(M, vrow, vcol)
        o.simplex()
        o.add_variable(3, 1.0, **flags)
        o.update_coefficient(1, 3, -2.0)
        o.simplex()
        picks.append((o.most_fractional()[0], o.is_integral()))
    assert picks == [(-1, True), (3, False), (3, False)]
    # the indices came from getNewElementIndex: branching cuts added later take fresh ones
    o.add_variable(9, 0.5)
    o.add_constraint(True, 4.0, 12, [(3, 1.0)])
    assert o.state().lastElementIndex == 13
    assert o.branch_and_cut().feasible


# ------------------------------------------------------------------ Model mirror -> index-level calls
class _RecordingLib:
    """The subset of libjslp_b200's C ABI the Model mirror's edits call, recording each call instead of touching a
    device.  It keeps the width, height and lastElementIndex the device reports through jslp_tab_info."""

    def __init__(self):
        self.calls, self.W, self.H, self.lei = [], 0, 0, 0

    def jslp_tab_create(self, ctx, W, H, cap, precision, out):
        out._obj.value = 1
        return 0

    def jslp_tab_upload(self, h, M, vrow, vcol, unres, n_index, ints, n_ints, n_opt, opt):
        return 0

    def jslp_tab_set_option(self, h, k, v):
        return 0

    def jslp_tab_destroy(self, h):
        return 0

    def jslp_tab_info(self, h, info):
        info[0], info[1], info[2], info[3], info[4], info[5] = self.W, self.H, 0, self.lei, 0, 0
        return 0

    def jslp_update_rhs(self, h, ci, d):
        self.calls.append(("update_rhs", ci, d))
        return 0

    def jslp_update_coefficient(self, h, ci, vi, d):
        self.calls.append(("update_coefficient", ci, vi, d))
        return 0

    def jslp_update_cost(self, h, vi, slot, d):
        self.calls.append(("update_cost", vi, slot, d))
        return 0

    def jslp_add_constraint(self, h, up, rhs, idx, tv, tc, n):
        terms = [] if n == 0 else list(zip((C.c_int32 * n).from_address(tv), (C.c_double * n).from_address(tc)))
        self.calls.append(("add_constraint", bool(up), rhs, idx, terms))
        self.H += 1
        self.lei = max(self.lei, idx + 1)
        return 0

    def jslp_remove_constraint(self, h, idx):
        self.calls.append(("remove_constraint", idx))
        self.H -= 1
        return 0

    def jslp_add_variable(self, h, idx, entry, slot, is_int, is_unres):
        self.calls.append(("add_variable", idx, entry, slot, bool(is_int), bool(is_unres)))
        self.W += 1
        self.lei = max(self.lei, idx + 1)
        return 0

    def jslp_remove_variable(self, h, idx):
        self.calls.append(("remove_variable", idx))
        self.W -= 1
        return 0


class _RecordingContext:
    def __init__(self):
        self.lib, self.handle = _RecordingLib(), 1


# A model with both senses of row, an Equality, and soft rows at two priorities (optional objectives 0 and 1).
EDIT_MODEL = {"optimize": "profit", "opType": "max",
              "constraints": {"wood": {"max": 300}, "labor": {"max": 110},
                              "storage": {"max": 400, "priority": "strong", "weight": 2},
                              "mix": {"equal": 4, "priority": "medium"},
                              "floor": {"min": 2}},
              "variables": {"table": {"wood": 30, "labor": 5, "profit": 1200, "storage": 30, "mix": 1, "floor": 1},
                            "dresser": {"wood": 20, "labor": 10, "profit": 1600, "storage": 50, "mix": -1, "floor": 1}}}


def edit_stages(m):
    """Model-level edits after a solve, in stages (a re-solve follows each).  Returns the stage callables."""
    byname = {}
    for c in m.constraints:
        byname.setdefault(c.name, []).append(c)
    wood, floor, storage = byname["wood"][0], byname["floor"][0], byname["storage"][0]
    mix_lo, mix_up = byname["mix"]
    from jslpsolver_b200.model import Equality
    mix = Equality(mix_up, mix_lo)
    table, dresser = [v for v in m.variables if v.id in ("table", "dresser")]
    r1 = storage.relaxation
    state = {}

    def stage1():
        wood.setRightHandSide(360)                       # upper bound: difference negated
        floor.setRightHandSide(3)                        # lower bound: difference as is
        m.setCost(1500, table)                           # maximisation: difference negated
        m.setCost(-3, r1)                                # a priority-1 variable: optional objective slot 0
        mix.setRightHandSide(5)                          # Equality: both rows

    def stage2():
        chair = state["chair"] = m.addVariable(700, "chair")
        bonus = state["bonus"] = m.addVariable(5, "bonus", priority="medium")
        mix.addTerm(1, chair)                            # Equality fans out: upper row, then lower row
        wood.addTerm(10, chair)
        storage.addTerm(12, bonus)
        extra = state["extra"] = m.smallerThan(25)
        for v in (table, dresser, chair):
            extra.addTerm(1, v)
        extra.addTerm(0.5, table)                        # an existing term: setVariableCoefficient(1.5)

    def stage3():
        m.removeConstraint(storage)                      # its relaxation variable goes too
        stool = m.addVariable(100, "stool")              # reuses the relaxation's index (last freed)
        state["low"] = m.greaterThan(1).addTerm(1, stool)  # reuses storage's index
        m.setCost(900, state["chair"])

    def stage4():
        m.removeConstraint(mix)                          # both rows; the shared relaxation variable once
        m.removeVariable(state["bonus"])

    return [stage1, stage2, stage3, stage4]


def record_edit_calls(model_json=EDIT_MODEL, stages=edit_stages):
    """The index-level calls the Model mirror makes for `stages`, stage by stage, on a recording tableau."""
    import jslpsolver_b200.tableau as T
    from jslpsolver_b200.model import Model

    class Recording(T.GpuTableau):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.context = _RecordingContext()

    orig = T.GpuTableau
    T.GpuTableau = Recording
    try:
        m = Model().loadJson(model_json)
    finally:
        T.GpuTableau = orig
    it = m.initial_tableau()
    lib = m.tableau.context.lib
    m.tableau.setModel(m)
    m.tableauInitialized = True
    lib.H, lib.W = it.matrix.shape
    lib.lei = lib.H + lib.W - 2
    out = []
    for stage in stages(m):
        lib.calls = []
        stage()
        out.append(lib.calls)
    return it, out


def test_model_edits_make_the_reference_index_level_calls():
    it, stages = record_edit_calls()
    # indices: wood 0, labor 1, storage 2, r1 3, mix >= 4, mix <= 5, r2 6, floor 7, table 8, dresser 9
    assert list(it.varIndexByRow) == [-1, 0, 1, 2, 4, 5, 7] and list(it.varIndexByCol) == [-1, 3, 6, 8, 9]
    assert it.optionalPriorities == [1, 2]
    assert stages[0] == [("update_rhs", 0, -60.0), ("update_rhs", 7, 1.0), ("update_cost", 8, -1, -300.0),
                         ("update_cost", 3, 0, 1.0), ("update_rhs", 5, -1.0), ("update_rhs", 4, 1.0)]
    assert stages[1] == [("add_variable", 10, 700.0, -1, False, False), ("add_variable", 11, 5.0, 1, False, False),
                         ("update_coefficient", 5, 10, -1.0), ("update_coefficient", 4, 10, 1.0),
                         ("update_coefficient", 0, 10, -10.0), ("update_coefficient", 2, 11, -12.0),
                         ("add_constraint", True, 25.0, 12, []),
                         ("update_coefficient", 12, 8, -1.0), ("update_coefficient", 12, 9, -1.0),
                         ("update_coefficient", 12, 10, -1.0), ("update_coefficient", 12, 8, -0.5)]
    assert stages[2] == [("remove_constraint", 2), ("remove_variable", 3), ("add_variable", 3, 100.0, -1, False, False),
                         ("add_constraint", False, 1.0, 2, []), ("update_coefficient", 2, 3, 1.0),
                         ("update_cost", 10, -1, -200.0)]
    assert stages[3] == [("remove_constraint", 5), ("remove_variable", 6), ("remove_constraint", 4),
                         ("remove_variable", 11)]


def test_minimisation_signs_and_flags():
    """Minimisation: setCost passes the difference as is and addVariable the negated cost; isInteger and
    isUnrestricted reach jslp_add_variable; a priority with no uploaded objective is refused on the host."""
    from jslpsolver_b200 import JslpError
    model = {"optimize": "cost", "opType": "min", "constraints": {"a": {"min": 3}, "b": {"max": 8}},
             "variables": {"x": {"cost": 2, "a": 1, "b": 1}, "y": {"cost": 3, "a": 1, "b": 2}}}

    def stages(m):
        x = m.variables[0]

        def s():
            m.setCost(5, x)
            m.addVariable(4, "z", isInteger=True)
            m.addVariable(-1, "w", isUnrestricted=True)
            with pytest.raises(JslpError, match="new priority"):
                m.addVariable(1, "soft", priority="weak")
        return [s]

    _, out = record_edit_calls(model, stages)
    calls = out[0]
    assert calls == [("update_cost", 2, -1, 3.0), ("add_variable", 4, -4.0, -1, True, False),
                     ("add_variable", 5, 1.0, -1, False, True)]

"""Irreducible infeasible subset (IIS) of an infeasible continuous LP: a set of constraint rows that is infeasible as a
whole and feasible once any one of them is dropped.  It answers "why is my model infeasible?".  The reference has no
counterpart; DESIGN.md section 2c is the contract.

Every membership test is phase 1 of the initial tableau restricted to a subset of its rows, run on the device in
batches (jslp_feasibility_batch: one CTA per set while the rows fit shared memory).  The rows tested come from the
sequential deletion filter; `deletion_filter` evaluates it speculatively, a batch at a time, and commits its decisions
in row order, so the answer is the one-row-at-a-time filter's.  Variable non-negativity is implicit in the tableau:
it is always kept and never reported."""
from __future__ import annotations

import numpy as np

FEASIBLE, INFEASIBLE, UNDECIDED = 0, 1, 2


def deletion_filter(test_batch, rows, width: int, prepass: bool = True):
    """The sequential deletion filter over `rows` (in order): for each row s, drop it if test(B minus s) is infeasible.

    `test_batch(sets)` takes a list of row lists and returns one verdict per list (FEASIBLE, INFEASIBLE or UNDECIDED;
    UNDECIDED keeps the row).  A round tests the next `width` steps at once, each on the set the filter will have
    reached if every earlier step of the round goes as predicted; the round commits steps in order and ends after the
    first step whose decision differs from its prediction.  The prediction is "keep", or with `prepass` (used only
    when width > 1) the verdict of one batch testing rows minus s for every s.  Every committed test is the one the
    literal filter makes, so the result does not depend on `width` or `prepass`.  Returns (kept rows, irreducible): irreducible is False when some
    row was kept on an UNDECIDED verdict."""
    rows = list(rows)
    n = len(rows)
    width = max(1, int(width))
    predict = [False] * n  # True = predicted delete
    if prepass and n > 1 and width > 1:
        verdicts = test_batch([rows[:i] + rows[i + 1:] for i in range(n)])
        predict = [v == INFEASIBLE for v in verdicts]
    deleted = [False] * n
    irreducible = True
    a = 0
    while a < n:
        ks = range(a, min(n, a + width))
        sets, spec = [], set()
        for k in ks:
            sets.append([rows[m] for m in range(n) if not deleted[m] and m not in spec and m != k])
            if predict[k]:
                spec.add(k)
        verdicts = test_batch(sets)
        for k, v in zip(ks, verdicts):
            deleted[k] = v == INFEASIBLE
            if v == UNDECIDED:
                irreducible = False
            a = k + 1
            if deleted[k] != predict[k]:
                break
    return [rows[m] for m in range(n) if not deleted[m]], irreducible


def certificate_support(M, vrow, vcol, precision, row_of_label) -> list:
    """Rows (initial row indices, sorted) behind the phase-1 certificate of the final tableau M of an infeasible test.
    The failing row r is phase 1's leaving-row rule on the final right-hand sides (lowest index with the minimum value
    below -precision).  Its support: every constraint whose slack is non-basic in a column c with |M[r,c]| > precision,
    plus the constraint whose slack is basic in row r.  `row_of_label` maps a slack's label to its initial row."""
    M = np.asarray(M, dtype=np.float64)
    rhs = M[1:, 0]
    r, best = 0, -precision
    for i, v in enumerate(rhs, start=1):
        if v < best:
            best, r = v, i
    if r == 0:
        raise ValueError("the final tableau has no row below -precision: it is not a phase-1 certificate")
    out = {row_of_label[int(vcol[c])] for c in range(1, M.shape[1])
           if int(vcol[c]) in row_of_label and abs(M[r, c]) > precision}
    if int(vrow[r]) in row_of_label:
        out.add(row_of_label[int(vrow[r])])
    return sorted(out)


def _check(solution) -> None:
    t = solution._tableau
    m = getattr(t, "model", None)
    if m is None:
        raise ValueError("iis() needs a solution of a Model (Solve(model, full=True) or Model.solve())")
    if m.getNumberOfIntegerVariables() > 0:
        raise ValueError("iis() is defined for continuous LPs only: the model has integer or binary variables")
    if any(c.relaxation is not None for c in m.constraints) or any(v.priority for v in m.variables):
        raise ValueError("iis() does not support soft constraints (weight / priority) or optional objectives")
    if solution.feasible:
        raise ValueError("iis() needs an infeasible solution: this LP is feasible")
    if solution._version != t._version or (t.handle is not None and t._solved_version != t._version):
        raise ValueError("iis() needs the model as this solution left it: the tableau was edited or solved again since")


def wave_width(context, height: int, width: int) -> int:
    """Sets one launch of the shared-memory batch runs at once: SMs x CTAs per SM, from the per-CTA shared memory of
    k_node_batch (node_smem_bytes in jslp_bnb.cuh, no cut rows).  1 when the rows do not fit shared memory: those
    tests run one after another, so speculating on them would only add work."""
    import torch
    p = torch.cuda.get_device_properties(context.device)
    ws = (width + 1) & ~1
    need = 8 * (height * ws + 2 * ws + height + 1) + 16 * height + 4 * (2 * height + width) + 16
    optin = getattr(p, "shared_memory_per_block_optin", 227 * 1024)
    per_sm = getattr(p, "shared_memory_per_multiprocessor", 228 * 1024)
    if need > optin - 4096:
        return 1
    return p.multi_processor_count * max(1, per_sm // (need + 2048))


def compute(solution, width=None, prepass=True) -> dict:
    """Solution.iis(): see the module docstring.  `width` / `prepass` tune the schedule only (None = one wave)."""
    from .tableau import GpuTableau
    _check(solution)
    t = solution._tableau
    m = t.model
    it = m.initial_tableau()
    H, W = it.matrix.shape
    rows = list(range(1, H))
    row_of_label = {int(it.varIndexByRow[r]): r for r in rows}
    scratch = GpuTableau(m.precision, context=t.context)  # the user's tableau is never touched
    lps = 0
    try:
        scratch.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted)
        scratch.save()
        scratch.phase1()  # test(all rows); a tableau without a model runs with the cycle check on
        lps += 1
        st = scratch.lastStatus
        if st.cycled:
            raise ValueError("iis(): phase 1 of the whole LP cycles, so its feasibility is undecided")
        if st.feasible:
            raise ValueError("iis(): the LP is feasible (presolve or the cycle check reported it infeasible)")
        support = certificate_support(scratch.matrix2d(), scratch.varIndexByRow, scratch.varIndexByCol,
                                      m.precision, row_of_label)
        scratch.restore()

        def test_batch(sets):
            nonlocal lps
            keep = np.zeros((len(sets), H), dtype=np.uint8)
            for i, s in enumerate(sets):
                keep[i, s] = 1
            keep[:, 0] = 1
            lps += len(sets)
            return [int(v) for v in scratch.feasibility_batch(keep)[0]]

        start = rows
        if support != rows and test_batch([support])[0] == INFEASIBLE:
            start = support
        K = wave_width(scratch.context, H, W) if width is None else width
        kept, irreducible = deletion_filter(test_batch, start, K, prepass)
    finally:
        scratch.close()
    constraints, names = [], []
    for r in kept:
        con = m.constraints[r - 1]
        name = con.name if con.name is not None else con.index
        constraints.append({"name": name, "type": "max" if con.isUpperBound else "min", "rhs": con.rhs})
        if name not in names:
            names.append(name)
    return {"constraints": constraints, "names": names, "irreducible": irreducible, "lps": lps}

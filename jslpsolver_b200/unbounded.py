"""Why a continuous LP is unbounded: the improving ray where the simplex stopped, a check of that claim, and an
irreducible set of variables whose caps make the LP bounded.  It answers "which direction runs away, is it real, and
what is the least I have to cap?".  The reference has no counterpart; DESIGN.md section 2l is the contract.

Every test is the recession-cone LP of the initial tableau (jslp_cone_create: column 0 set to +0 plus the
normalisation row sum_j d_j <= 1) with the columns of the capped variables set to +0, solved on the device in batches
(jslp_column_batch).  The LP with caps on S is bounded exactly when that cone LP ends at M[0,0] == 0 (within the
precision).  The additive phase grows S by the support of each ray it finds; `iis.deletion_filter` then removes every
variable whose cap is not needed, in column order, so the answer is the one-variable-at-a-time filter's."""
from __future__ import annotations

import numpy as np

from . import iis

RAY, BOUNDED, UNDECIDED = 0, 1, 2
COL_OPTIMAL, COL_UNBOUNDED, COL_CYCLED, COL_INFEASIBLE = 0, 1, 2, 3


def _check(solution) -> None:
    t = solution._tableau
    m = getattr(t, "model", None)
    if m is None:
        raise ValueError("unbounded() needs a solution of a Model (Solve(model, full=True) or Model.solve())")
    if m.getNumberOfIntegerVariables() > 0:
        raise ValueError("unbounded() is defined for continuous LPs only: the model has integer or binary variables")
    if any(c.relaxation is not None for c in m.constraints) or any(v.priority for v in m.variables):
        raise ValueError("unbounded() does not support soft constraints (weight / priority) or optional objectives")
    if m.unrestrictedVariables:
        raise ValueError("unbounded() does not support unrestricted variables: the ray would be two-sided")
    if not solution.feasible:
        raise ValueError("unbounded() needs an unbounded solution: this LP is infeasible")
    if solution.bounded:
        raise ValueError("unbounded() needs an unbounded solution: this LP is bounded")
    if solution._version != t._version or (t.handle is not None and t._solved_version != t._version):
        raise ValueError("unbounded() needs the model as this solution left it: the tableau was edited or solved again "
                         "since")


def verdict(status: int, eval_raw: float, precision: float) -> int:
    """RAY when the cone LP improves (|M[0,0]| > P, or phase 2 stopped unbounded), BOUNDED when it does not, UNDECIDED
    when its cycle check fired (or, for a tableau that is not a cone, phase 1 found it infeasible)."""
    if status == COL_CYCLED or status == COL_INFEASIBLE:
        return UNDECIDED
    if status == COL_UNBOUNDED or abs(eval_raw) > precision:
        return RAY
    return BOUNDED


def support(rhs, vrow, col_of_label, precision) -> list:
    """Columns (sorted) of the structural variables basic in a final cone tableau with value > precision."""
    return sorted(col_of_label[int(vrow[r])] for r in range(1, len(vrow))
                  if int(vrow[r]) in col_of_label and rhs[r] > precision)


def ray_report(m, it, rhs, vrow, vcol, entering, column, precision) -> dict:
    """The ray, rate, point, per-row rates and blocking rows of the stop tableau (column 0 `rhs`, labels `vrow` /
    `vcol`, the entering label and its column `column`), against the initial tableau `it` of model `m`."""
    var_of = {v.index: v for v in m.variables}
    rate_of, value_of = {int(entering): 1.0}, {}
    for r in range(1, len(vrow)):
        lab = int(vrow[r])
        if lab in var_of:
            rate_of[lab] = -float(column[r]) + 0.0
            value_of[lab] = float(rhs[r])
    ray = {v.id: rate_of[v.index] for v in m.variables if rate_of.get(v.index, 0.0) != 0.0}
    point = {v.id: value_of[v.index] for v in m.variables if value_of.get(v.index, 0.0) != 0.0}
    rate = 0.0
    for v in m.variables:
        rate += float(v.cost) * rate_of.get(v.index, 0.0)
    W = it.matrix.shape[1]
    x, d = np.zeros(W - 1), np.zeros(W - 1)
    for c in range(1, W):
        x[c - 1] = value_of.get(int(it.varIndexByCol[c]), 0.0)
        d[c - 1] = rate_of.get(int(it.varIndexByCol[c]), 0.0)
    constraints, blocking = [], []
    for r in range(1, it.matrix.shape[0]):
        con = m.constraints[r - 1]
        a = (1.0 if con.isUpperBound else -1.0) * it.matrix[r, 1:]
        name = con.name if con.name is not None else con.index
        act, rr = float(a @ x) + 0.0, float(a @ d) + 0.0
        constraints.append({"name": name, "type": "max" if con.isUpperBound else "min", "rhs": con.rhs,
                            "activity": act, "rate": rr})
        if ((con.isUpperBound and rr > precision) or (not con.isUpperBound and rr < -precision)) \
                and name not in blocking:
            blocking.append(name)
    if (-rate if m.isMinimization else rate) <= precision:
        blocking.append("objective")
    return {"ray": ray, "rate": rate, "point": point, "constraints": constraints, "blocking": blocking}


def bounding_set(test_batch, n_columns: int, width: int, prepass: bool = True):
    """The two phases over a cone test.  `test_batch(sets)` takes lists of capped columns and returns one (verdict,
    support) per list.  Returns (confirmed, columns, irreducible): confirmed is None when the first test is undecided;
    columns is None when the additive phase is undecided (or a ray has no support above the precision)."""
    S: list = []
    confirmed = None
    for _ in range(n_columns + 1):
        v, sup = test_batch([S])[0]
        if confirmed is None and not S:
            if v == UNDECIDED:
                return None, None, False
            confirmed = v == RAY
            if not confirmed:
                return False, [], True
        if v == BOUNDED:
            break
        if v == UNDECIDED or not sup:
            return confirmed, None, False
        S = sorted(set(S) | set(sup))
    else:
        return confirmed, None, False
    # "caps on B minus s still bound the LP" plays the role of INFEASIBLE in the row filter
    mapped = {BOUNDED: iis.INFEASIBLE, RAY: iis.FEASIBLE, UNDECIDED: iis.UNDECIDED}
    kept, irreducible = iis.deletion_filter(lambda sets: [mapped[v] for v, _ in test_batch(sets)], S, width, prepass)
    return confirmed, kept, irreducible


def compute(solution, width=None, prepass=True) -> dict:
    """Solution.unbounded(): see the module docstring.  `width` / `prepass` tune the schedule only (None = one wave)."""
    from .tableau import GpuTableau
    _check(solution)
    t = solution._tableau
    m = t.model
    P = m.precision
    it = m.initial_tableau()
    H, W = it.matrix.shape
    # the stop tableau: column 0, the labels and the entering column only
    vrow, vcol = t.varIndexByRow, t.varIndexByCol
    entering = t.unboundedVarIndex
    cstar = [c for c in range(1, len(vcol)) if int(vcol[c]) == entering]
    if entering is None or not cstar:
        raise ValueError("unbounded(): the solution does not name the entering variable of its stop")
    out = ray_report(m, it, t.rhs_column(), vrow, vcol, entering, t.column(cstar[0]), P)
    structural = {v.index for v in m.variables}
    col_of_label = {int(it.varIndexByCol[c]): c for c in range(1, W) if int(it.varIndexByCol[c]) in structural}
    scratch = GpuTableau(P, context=t.context)  # the user's tableau is never touched
    cone = None
    lps = 0
    try:
        scratch.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted)
        cone = scratch.cone()
        cone.save()

        def test_batch(sets):
            nonlocal lps
            keep = np.ones((len(sets), W), dtype=np.uint8)
            for i, s in enumerate(sets):
                keep[i, list(s)] = 0
            keep[:, 0] = 1
            lps += len(sets)
            res = cone.column_batch(keep)
            return [(verdict(int(res["status"][i]), float(res["eval_raw"][i]), P),
                     support(res["rhs"][i], res["vrow"][i], col_of_label, P)) for i in range(len(sets))]

        K = iis.wave_width(cone.context, H + 1, W) if width is None else width
        confirmed, cols, irreducible = bounding_set(test_batch, len(col_of_label), K, prepass)
    finally:
        if cone is not None:
            cone.close()
        scratch.close()
    label_of = {c: lab for lab, c in col_of_label.items()}
    if cols is None:
        bound = None
    else:
        ids = {label_of[c] for c in cols}
        bound = {"variables": [v.id for v in m.variables if v.index in ids], "irreducible": irreducible}
    out.update(confirmed=confirmed, bound=bound, lps=lps)
    return out

"""oracle/warmstart.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The definition of a warm start (DESIGN.md section 2f) over the C oracle: the tableau Model.solve() uploads, the crash
of the saved basis with OracleTableau.pivot (the reference's Tableau.pivot) and NumPy selection, then simplex() with
the model's cycle check, shaped as Solve() shapes a result.  The names of the basis are resolved by the package's own
pure-host plan() on a host Model of the same JSON, which numbers variables and rows as ref_model.RefModel does."""
from __future__ import annotations

import numpy as np

from . import ref_model

REJECTED, BASIC = -1, -2


def crash(tab, enter, leave, precision):
    """The crash on OracleTableau `tab`: (records n x 4, pivots).  A record is (label, row, column, leaving label) of
    a pivot, (label, row, -1, BASIC) for a label already basic, (label, -1, column, REJECTED) when no row is eligible."""
    records, n = [], 0
    for lab in (int(x) for x in enter):
        vrow, vcol = tab.maps()
        rows = np.nonzero(vrow[1:] == lab)[0]
        if len(rows):
            records.append((lab, 1 + int(rows[0]), -1, BASIC))
            continue
        cols = np.nonzero(vcol[1:] == lab)[0]
        if not len(cols):
            records.append((lab, -1, -1, REJECTED))
            continue
        c = 1 + int(cols[0])
        col = tab.matrix()[1:, c]
        labels = vrow[1:].astype(np.int64)
        ok = (labels >= 0) & (labels < len(leave))
        gives_up = np.zeros(len(labels), dtype=bool)
        gives_up[ok] = np.asarray(leave)[labels[ok]] != 0
        with np.errstate(invalid="ignore"):
            eligible = gives_up & ((col < -precision) | (precision < col))
        if not eligible.any():
            records.append((lab, -1, c, REJECTED))
            continue
        r = 1 + int(np.argmax(np.where(eligible, np.abs(col), -1.0)))  # first maximum: lowest row on ties
        records.append((lab, r, c, int(vrow[r])))
        tab.pivot(r, c)
        n += 1
    return np.asarray(records, dtype=np.int32).reshape(-1, 4), n


def host_model(jm, precision=None):
    """The package's host Model of jm, without a device tableau (for plan() and basis_of())."""
    from jslpsolver_b200.model import Model
    return Model(precision).loadJson(jm)


def warm_solve(jm, basis, precision=None, fast_cycles=True, pivot_log=0):
    """Solve(jm, precision, full=True, basis=basis) restated: (OracleSolution, crash records, crash pivots, unknown).
    A model presolve declares infeasible returns before any tableau exists (records None)."""
    from jslpsolver_b200.warmstart import plan
    enter, leave, unknown = plan(host_model(jm, precision), basis)
    model = ref_model.RefModel(precision).loadJson(jm)
    sol = ref_model.OracleSolution()
    sol.model = model
    if model.usePresolve:
        infeasible, fixed = ref_model.presolve(model)
        if infeasible:
            sol.feasible = False
            sol.evaluation = 0.0 if model.isMinimization else -0.0
            return sol, None, 0, unknown
        for var in fixed:
            var.value = fixed[var]
            var.cost = 0
    M, vrow, vcol, _, _ = model.build_tableau()
    unres = np.zeros(M.shape[0] + M.shape[1] - 2, dtype=np.uint8)
    for i in model.unrestrictedVariables:
        unres[i] = 1
    tab = ref_model.OracleTableau(M, vrow, vcol, precision=model.precision, unrestricted=unres,
                                  check_cycles=model.checkForCycles, fast_cycles=fast_cycles,
                                  is_min=model.isMinimization, pivot_log=pivot_log)
    records, n = crash(tab, enter, leave, model.precision)
    st = tab.simplex()
    sol.tableau, sol.state = tab, st
    sol.feasible, sol.bounded = bool(st.feasible), bool(st.bounded)
    sol.evaluation = st.evaluation if model.isMinimization else -st.evaluation
    rounding = ref_model.js_round(1 / model.precision)
    Mx = tab.matrix()
    vrow_f, _ = tab.maps()
    for r in range(1, st.height):  # generateSolutionSet, solution.ts:35-60
        var = model.variablesPerIndex.get(int(vrow_f[r]))
        if var is None or var.isSlack:
            continue
        sol.solutionSet[var.id] = ref_model.js_round((ref_model.EPSILON + Mx[r, 0]) * rounding) / rounding
    return sol, records, n, unknown


def basis(jm, sol, precision=None) -> dict:
    """Solution.basis() of the oracle solution `sol` of jm."""
    from jslpsolver_b200.warmstart import basis_of
    vrow, _ = sol.tableau.maps()
    return basis_of(host_model(jm, precision), vrow)

"""oracle/scenarios.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The definition of Solution.scenarios() (DESIGN.md section 2e) over the C oracle: every scenario starts from an
OracleTableau of the solved state, applies its edits in order with update_rhs / update_cost (dynamic-modification.ts),
runs simplex() with the model's cycle check and is shaped as Solve() shapes a result (generateSolutionSet +
ref_model.simplify).  Edits are (kind, index, difference) triples: kind 0 = right-hand side of the constraint with that
slack index, kind 1 = cost of that variable."""
from __future__ import annotations

import numpy as np

from . import ref_model


def run(sol, edits):
    """One scenario from the solved oracle solution `sol` (ref_model.solve_full): (final state, the oracle tableau)."""
    model = sol.model
    M = sol.tableau.matrix()
    vrow, vcol = sol.tableau.maps()
    unres = np.zeros(M.shape[0] + M.shape[1] - 2, dtype=np.uint8)
    for i in model.unrestrictedVariables:
        unres[i] = 1
    tab = ref_model.OracleTableau(M, vrow, vcol, precision=model.precision, unrestricted=unres,
                                  check_cycles=model.checkForCycles, fast_cycles=True, is_min=model.isMinimization)
    for kind, index, difference in edits:
        if kind == 0:
            tab.update_rhs(index, difference)
        else:
            tab.update_cost(index, difference)
    return tab.simplex(), tab


def result(sol, edits) -> dict:
    """The Solve() result of one scenario."""
    st, tab = run(sol, edits)
    model = sol.model
    out = ref_model.OracleSolution()
    out.feasible, out.bounded = bool(st.feasible), bool(st.bounded)
    # simplex() leaves Tableau.evaluation alone when it ends infeasible or in a cycle: the solved tableau's evaluation
    # stands (a fresh oracle tableau would start from 0)
    out.evaluation = (st.evaluation if model.isMinimization else -st.evaluation) if st.feasible else sol.evaluation
    rounding = ref_model.js_round(1 / model.precision)
    Mx = tab.matrix()
    vrow, _ = tab.maps()
    for r in range(1, st.height):  # generateSolutionSet, solution.ts:35-60
        var = model.variablesPerIndex.get(int(vrow[r]))
        if var is None or var.isSlack:
            continue
        out.solutionSet[var.id] = ref_model.js_round((ref_model.EPSILON + Mx[r, 0]) * rounding) / rounding
    return ref_model.simplify(out)

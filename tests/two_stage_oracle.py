"""The restatement of TwoStage() (DESIGN.md section 2u) over the C oracle -- TEST INFRASTRUCTURE.

It replaces the two device steps of the L-shaped loop and keeps the host bookkeeping (two_stage.run), so a device run can
be matched iteration for iteration:
- the master: ref_model.solve_full of the master JSON, the oracle's Solve() (presolve is off in the JSON);
- the recourse tableau: the recourse model's initial tableau solved on an OracleTableau, or left as built when that
  solve does not end optimal;
- each batch: per case, an OracleTableau of that tableau with the case's edits applied in order (update_rhs /
  update_cost) and simplex() with the cycle check on, as Solution.scenarios() is defined; then the certificate row
  (row 0 at an optimum, the first most negative column-0 entry below -precision when infeasible), its multipliers of
  the recourse rows through the final labels, and alpha summed over the rows in increasing order."""
from __future__ import annotations

import math

import numpy as np

from jslpsolver_b200.model import Model
from jslpsolver_b200.scenarios import CYCLED, INFEASIBLE, OPTIMAL, UNBOUNDED
from jslpsolver_b200 import two_stage
from oracle import ref_model


def status_of(st) -> int:
    return CYCLED if st.cyclePhase else INFEASIBLE if not st.feasible else UNBOUNDED if not st.bounded else OPTIMAL


def cert_row(status: int, col0, precision: float) -> int:
    if status == OPTIMAL:
        return 0
    if status != INFEASIBLE:
        return -1
    r0, v = -1, -precision
    for r in range(1, len(col0)):
        if col0[r] < v:
            r0, v = r, col0[r]
    return r0


def multipliers(status, M, vrow, vcol, rows, precision) -> list:
    """u[i]: the certificate row's multiplier of the row whose slack label is rows[i]."""
    u = [0.0] * len(rows)
    cr = cert_row(status, M[:, 0], precision)
    if cr < 0:
        return u
    pos = {label: i for i, label in enumerate(rows)}
    for c in range(1, M.shape[1]):
        if int(vcol[c]) in pos:
            u[pos[int(vcol[c])]] = float(M[cr, c])
    for r in range(1, M.shape[0]):
        if int(vrow[r]) in pos:
            u[pos[int(vrow[r])]] = 1.0 if r == cr else 0.0
    return u


def alpha_of(u, tech) -> list:
    """alpha[j] = sum_i u[i] * tech[i][j] over i in increasing order, unfused."""
    out = []
    for j in range(tech.shape[1] if tech.ndim == 2 else 0):
        acc = 0.0
        for i in range(len(u)):
            acc = acc + u[i] * float(tech[i, j])
        out.append(acc)
    return out


class Oracle:
    """The backend of two_stage.run over the C oracle."""

    def __init__(self, precision=None):
        self.precision = precision
        self.base = None

    def launches(self) -> int:
        return 0

    def master(self, jm):
        sol = ref_model.solve_full(jm, self.precision, fast_cycles=True)
        st = sol.state
        status = status_of(st)
        values = {}
        M = sol.tableau.matrix()
        if status == OPTIMAL:
            vrow, _ = sol.tableau.maps()
            for r in range(1, st.height):
                var = sol.model.variablesPerIndex.get(int(vrow[r]))
                if var is not None and not var.isSlack:
                    values[var.id] = float(M[r, 0])
        return status, float(M[0, 0]) if status == OPTIMAL else math.nan, values, int(st.lastP1 + st.lastP2)

    def _tableau(self, M, vrow, vcol):
        return ref_model.OracleTableau(M, vrow, vcol, precision=self.m.precision, check_cycles=True, fast_cycles=True,
                                       is_min=self.m.isMinimization)

    def recourse(self, jm):
        m = Model(self.precision).loadJson(jm)
        self.m = m
        it = m.initial_tableau()
        tab = self._tableau(it.matrix, it.varIndexByRow, it.varIndexByCol)
        st = tab.simplex()
        if status_of(st) == OPTIMAL:
            vrow, vcol = tab.maps()
            self.base = (tab.matrix().copy(), vrow.copy(), vcol.copy())
        else:
            self.base = (it.matrix.copy(), it.varIndexByRow.copy(), it.varIndexByCol.copy())
        return m, int(st.lastP1 + st.lastP2)

    def case(self, edits, rows, tech):
        """One case: (status, eval_raw, p1, p2, column 0, row labels, cert_rhs, alpha)."""
        tab = self._tableau(*self.base)
        for kind, index, difference in edits:
            if kind == 0:
                tab.update_rhs(index, difference)
            else:
                tab.update_cost(index, difference)
        st = tab.simplex()
        status = status_of(st)
        M = tab.matrix()
        vrow, vcol = tab.maps()
        u = multipliers(status, M, vrow, vcol, rows, self.m.precision)
        cr = cert_row(status, M[:, 0], self.m.precision)
        return (status, float(M[0, 0]), int(st.lastP1), int(st.lastP2), M[:, 0].copy(), vrow.copy(),
                float(M[cr, 0]) if cr >= 0 else math.nan, alpha_of(u, tech))

    def batch(self, edits, offsets, rows, tech):
        n = len(offsets) - 1
        per_case = tech.ndim == 3
        res = [self.case(edits[offsets[s]:offsets[s + 1]], rows, tech[s] if per_case else tech) for s in range(n)]
        n_first = tech.shape[-1]
        return {"status": np.array([r[0] for r in res], dtype=np.int32),
                "eval_raw": np.array([r[1] for r in res], dtype=np.float64),
                "p1": np.array([r[2] for r in res], dtype=np.int32),
                "p2": np.array([r[3] for r in res], dtype=np.int32),
                "rhs": np.array([r[4] for r in res], dtype=np.float64),
                "vrow": np.array([r[5] for r in res], dtype=np.int32),
                "cert_rhs": np.array([r[6] for r in res], dtype=np.float64),
                "alpha": np.array([r[7] for r in res], dtype=np.float64).reshape(n, n_first)}

    def close(self):
        pass


def TwoStage(model, cases, first, probabilities=None, **kw) -> dict:
    """TwoStage() with the device steps restated over the C oracle."""
    return two_stage.TwoStage(None, model, cases, first, probabilities, backend=Oracle(kw.get("precision")), **kw)

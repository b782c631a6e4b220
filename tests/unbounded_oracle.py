"""tests/unbounded_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The definition of Solution.unbounded() (DESIGN.md section 2l) in NumPy over the C oracle: the cone tableau of an initial
tableau (rule 1), one cone test as ref_model.OracleTableau's simplex (cycle check on) of a NumPy copy with the capped
columns set to +0 (rule 2), and the literal additive and one-column-at-a-time deletion filters, with no batching or
speculation (rule 3).  The stop tableau comes from the same oracle's simplex of the model's initial tableau."""
from __future__ import annotations

import numpy as np

import lexicographic_oracle as LO
from oracle import ref_model

RAY, BOUNDED, UNDECIDED = 0, 1, 2
OPTIMAL, INFEASIBLE, UNBOUNDED, CYCLED = LO.OPTIMAL, LO.INFEASIBLE, LO.UNBOUNDED, LO.CYCLED


def cone(M, vrow, vcol, label):
    """Rule 1: (K, vrow', vcol') -- M's rows with column 0 set to +0, then the row sum_j d_j <= 1."""
    M = np.ascontiguousarray(M, dtype=np.float64)
    H, W = M.shape
    K = np.zeros((H + 1, W), dtype=np.float64)
    K[:H] = M
    K[:H, 0] = 0.0
    K[H, :] = 1.0
    vr = np.concatenate([np.asarray(vrow, dtype=np.int32), [label]]).astype(np.int32)
    return K, vr, np.asarray(vcol, dtype=np.int32).copy()


def solve(K, vrow, vcol, precision, capped):
    """Rule 2: (status, pivots, final tableau, row labels) of the cone with the columns `capped` set to +0."""
    Kc = np.array(K, dtype=np.float64)
    if len(capped):
        Kc[:, list(capped)] = 0.0
    status, p1, p2, Mx, vr, _ = LO.solve(Kc, vrow, vcol, precision)
    return status, p1 + p2, Mx, vr


def test(K, vrow, vcol, precision, capped, structural_cols):
    """(verdict, support columns, status, eval_raw, pivots, final column 0, final row labels) of one cone test."""
    status, piv, Mx, vr = solve(K, vrow, vcol, precision, capped)
    if status in (CYCLED, INFEASIBLE):
        v = UNDECIDED
    elif status == UNBOUNDED or abs(Mx[0, 0]) > precision:
        v = RAY
    else:
        v = BOUNDED
    col_of = {int(vcol[c]): c for c in structural_cols}
    sup = sorted(col_of[int(vr[r])] for r in range(1, len(vr)) if int(vr[r]) in col_of and Mx[r, 0] > precision)
    return v, sup, status, float(Mx[0, 0]), piv, Mx[:, 0].copy(), vr


def bound(K, vrow, vcol, precision, structural_cols):
    """Rule 3: (confirmed, capped columns or None, irreducible, lps)."""
    lps = 0

    def t(S):
        nonlocal lps
        lps += 1
        return test(K, vrow, vcol, precision, S, structural_cols)[:2]

    S = []
    v, sup = t(S)
    if v == UNDECIDED:
        return None, None, False, lps
    if v == BOUNDED:
        return False, [], True, lps
    while v == RAY:
        if not sup:
            return True, None, False, lps
        S = sorted(set(S) | set(sup))
        v, sup = t(S)
    if v == UNDECIDED:
        return True, None, False, lps
    B, irreducible = list(S), True
    for s in S:
        v, _ = t([x for x in B if x != s])
        if v == BOUNDED:
            B.remove(s)
        elif v == UNDECIDED:
            irreducible = False
    return True, B, irreducible, lps


def stop_tableau(it, precision, check_cycles=True):
    """The oracle's simplex of the initial tableau: (final tableau, row labels, column labels, state)."""
    tab = ref_model.OracleTableau(it.matrix, it.varIndexByRow, it.varIndexByCol, precision=precision,
                                  unrestricted=it.unrestricted, check_cycles=check_cycles, fast_cycles=True)
    st = tab.simplex()
    vr, vc = tab.maps()
    return tab.matrix(), vr, vc, st


def unbounded(m):
    """Solution.unbounded() over the oracle for a Model `m` (presolve already applied as Model.solve applies it), or
    None when the oracle's simplex does not stop unbounded."""
    from jslpsolver_b200.unbounded import ray_report
    P = m.precision
    it = m.initial_tableau()
    F, vr, vc, st = stop_tableau(it, P, m.checkForCycles)
    if not st.feasible or st.bounded:
        return None
    cstar = [c for c in range(1, len(vc)) if int(vc[c]) == int(st.unboundedVar)][0]
    out = ray_report(m, it, F[:, 0], vr, vc, int(st.unboundedVar), F[:, cstar], P)
    H, W = it.matrix.shape
    structural = {v.index for v in m.variables}
    cols = [c for c in range(1, W) if int(it.varIndexByCol[c]) in structural]
    K, kvr, kvc = cone(it.matrix, it.varIndexByRow, it.varIndexByCol, W + H - 2)
    confirmed, B, irreducible, lps = bound(K, kvr, kvc, P, cols)
    if B is None:
        out["bound"] = None
    else:
        ids = {int(it.varIndexByCol[c]) for c in B}
        out["bound"] = {"variables": [v.id for v in m.variables if v.index in ids], "irreducible": irreducible}
    out.update(confirmed=confirmed, lps=lps)
    return out


def presolved_model(jm, precision=None):
    """Model.loadJson(jm) with presolve applied as Model.solve applies it (fixed variables get cost 0), on the CPU."""
    from jslpsolver_b200.model import Model, presolve
    m = Model(precision).loadJson(jm)
    if m.usePresolve:
        m.presolveResult = presolve(m)
        for variable, value in m.presolveResult.fixedVariables.items():
            variable.value = value
            variable.cost = 0
    return m

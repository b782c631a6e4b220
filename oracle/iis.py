"""oracle/iis.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restatement of the IIS contract (DESIGN.md section 2c) over the C oracle: `test` is the reference's phase 1
(simplex.ts:25-98, cycle check on) on cost row 0 plus a subset of the initial tableau's rows, `start_set` the
certificate start set S0 and `literal_filter` the one-row-at-a-time deletion filter, with no batching or speculation.

orc_upload needs labels below W + H - 2, so the kept rows' labels are relabelled densely in their order; phase 1 reads
labels only for the unrestricted flag and the cycle check, and an injective relabel changes neither."""
from __future__ import annotations

import numpy as np

from . import ref_model

FEASIBLE, INFEASIBLE, UNDECIDED = 0, 1, 2


def _phase1(M, vrow, vcol, unres, precision, rows):
    """(verdict, pivots, final tableau, final labels in the original numbering) of phase 1 on rows 0 + `rows`."""
    M = np.asarray(M, dtype=np.float64)
    keep = [0] + sorted(rows)
    Ms = np.ascontiguousarray(M[keep])
    labels = sorted(set(int(v) for v in np.asarray(vrow)[keep[1:]]) | set(int(v) for v in np.asarray(vcol)[1:]))
    new = {old: i for i, old in enumerate(labels)}
    vr = np.array([-1] + [new[int(vrow[r])] for r in keep[1:]], dtype=np.int32)
    vc = np.array([-1] + [new[int(v)] for v in np.asarray(vcol)[1:]], dtype=np.int32)
    u = np.array([1 if (unres is not None and old < len(unres) and unres[old]) else 0 for old in labels], dtype=np.uint8)
    tab = ref_model.OracleTableau(Ms, vr, vc, precision=precision, unrestricted=u, check_cycles=True, fast_cycles=True)
    pivots = int(tab.phase1())
    st = tab.state()
    verdict = UNDECIDED if st.cyclePhase == 1 else (FEASIBLE if st.feasible else INFEASIBLE)
    fr, fc = tab.maps()
    back = lambda a: np.array([-1 if v < 0 else labels[v] for v in a], dtype=np.int64)
    return verdict, pivots, tab.matrix(), back(fr), back(fc)


def test(M, vrow, vcol, unres, precision, rows):
    """(verdict, phase-1 pivots) of test(rows)."""
    v, p, _, _, _ = _phase1(M, vrow, vcol, unres, precision, rows)
    return v, p


def start_set(M, vrow, vcol, unres, precision):
    """(S0, support, whole-LP verdict): S0 is the certificate support when it tests infeasible, else every row;
    S0 is None unless the whole LP tests infeasible."""
    H = np.asarray(M).shape[0]
    rows = list(range(1, H))
    v, _, F, fr, fc = _phase1(M, vrow, vcol, unres, precision, rows)
    if v != INFEASIBLE:
        return None, None, v
    row_of = {int(vrow[r]): r for r in rows}
    rhs = F[1:, 0]
    r = 1 + int(np.argmin(rhs))  # lowest index of the minimum; it is below -precision in an infeasible final tableau
    assert rhs[r - 1] < -precision
    support = sorted({row_of[int(fc[c])] for c in range(1, F.shape[1]) if int(fc[c]) in row_of and abs(F[r, c]) > precision}
                     | ({row_of[int(fr[r])]} if int(fr[r]) in row_of else set()))
    if support != rows and test(M, vrow, vcol, unres, precision, support)[0] == INFEASIBLE:
        return support, support, v
    return rows, support, v


def literal_filter(M, vrow, vcol, unres, precision, S0):
    """(kept rows, irreducible) of B = S0; for s in S0: if test(B minus s) is infeasible, B = B minus s."""
    B = list(S0)
    irreducible = True
    for s in list(S0):
        v, _ = test(M, vrow, vcol, unres, precision, [x for x in B if x != s])
        if v == INFEASIBLE:
            B.remove(s)
        elif v == UNDECIDED:
            irreducible = False
    return B, irreducible


def iis(it, precision):
    """(kept rows, irreducible, S0 was the support) for an InitialTableau `it` whose LP tests infeasible; None else."""
    M, vrow, vcol, unres = it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted
    S0, support, _ = start_set(M, vrow, vcol, unres, precision)
    if S0 is None:
        return None
    kept, irreducible = literal_filter(M, vrow, vcol, unres, precision, S0)
    return kept, irreducible, S0 == support

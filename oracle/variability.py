"""oracle/variability.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The definition of Solution.variability() (DESIGN.md section 2h) in NumPy over the C oracle: the face tableau of a final
tableau (rules 1 and 2), one target LP on it (rule 3: the one-edit cost scenario of oracle/scenarios.py with the cycle
check on), and the ranges of a list of labels with the LPs rule 4 leaves out (rules 4 and 5)."""
from __future__ import annotations

import math
import types

import numpy as np

from . import scenarios as OS

OPTIMAL, INFEASIBLE, UNBOUNDED, CYCLED = 0, 1, 2, 3


def face(M, vcol, precision):
    """(map, F, vcol') of the final tableau M: rules 1 and 2 (F at its logical width, without the stride padding)."""
    M = np.asarray(M, dtype=np.float64)
    kept = [0] + [c for c in range(1, M.shape[1]) if M[0, c] >= -precision and M[0, c] <= precision]
    F = M[:, kept].copy()
    F[0, :] = 0.0
    return np.array(kept, dtype=np.int32), F, np.asarray(vcol, dtype=np.int32)[kept].copy()


def target(F, vrow, vcol_f, precision, label, sense):
    """Rule 3 for `label` and sense +1 (maximise) / -1 (minimise): (status, eval_raw, phase-1 pivots, phase-2 pivots,
    final column 0, final row labels).

    The C oracle sizes its label maps from the shape of the tableau it is given, and F keeps the labels of the wider
    parent, so the labels are renamed to their rank among F's labels for the run and named back afterwards.  The order
    of the labels is kept, no variable is unrestricted or integer here, and nothing else in the simplex reads a
    label's value."""
    vrow, vcol_f = np.asarray(vrow, dtype=np.int32), np.asarray(vcol_f, dtype=np.int32)
    present = np.array(sorted([int(v) for v in vrow[1:]] + [int(v) for v in vcol_f[1:]]), dtype=np.int32)
    rank = {int(v): k for k, v in enumerate(present)}
    rename = lambda a: np.array([-1] + [rank[int(v)] for v in a[1:]], dtype=np.int32)  # noqa: E731
    model = types.SimpleNamespace(precision=precision, unrestrictedVariables={}, checkForCycles=True,
                                  isMinimization=True)
    src = types.SimpleNamespace(model=model, tableau=types.SimpleNamespace(
        matrix=lambda: F, maps=lambda: (rename(vrow), rename(vcol_f))))
    st, tab = OS.run(src, [(1, rank[int(label)], -float(sense))])
    Mx, (vr, _) = tab.matrix(), tab.maps()
    status = CYCLED if st.cyclePhase else INFEASIBLE if not st.feasible else UNBOUNDED if not st.bounded else OPTIMAL
    back = np.array([-1] + [int(present[v]) for v in vr[1:]], dtype=np.int32)
    return status, float(Mx[0, 0]), int(st.lastP1), int(st.lastP2), Mx[:, 0].copy(), back


def end(status, eval_raw, sense):
    """The range end a target LP gives: -s * eval_raw (a zero of either sign reads +0), s * inf, or None."""
    if status == OPTIMAL:
        return -sense * eval_raw + 0.0
    return sense * math.inf if status == UNBOUNDED else None


def ranges(M, vrow, vcol, precision, labels):
    """Rules 3 to 5 for `labels` on the final tableau (M, vrow, vcol): ({label: {"value", "min", "max", "argmin",
    "argmax"}}, free, lps, the submitted (label, sense) list in order).  argmin / argmax are (column 0, row labels) of
    the vertex reached, the final tableau's own where no LP runs, None where the LP gave no answer."""
    M = np.asarray(M, dtype=np.float64)
    kept, F, vcol_f = face(M, vcol, precision)
    row_of = {int(vrow[r]): r for r in range(1, len(vrow))}
    col_of = {int(vcol[c]): c for c in range(1, len(vcol))}
    here = (M[:, 0].copy(), np.asarray(vrow, dtype=np.int32).copy())
    out, submitted = {}, []
    for lab in labels:
        r = row_of.get(int(lab))
        value = float(M[r, 0]) if r is not None else 0.0
        e = {"value": value, "min": value, "max": value, "argmin": here, "argmax": here}
        senses = []
        if len(kept) > 1:
            if r is not None:
                senses = [-1, 1]
            elif col_of[int(lab)] in set(int(c) for c in kept):
                senses = [1]
        for s in senses:
            status, ev, _, _, rhs, vr = target(F, vrow, vcol_f, precision, lab, s)
            submitted.append((int(lab), s))
            side = "max" if s > 0 else "min"
            e[side] = end(status, ev, s)
            e["arg" + side] = (rhs, vr) if status == OPTIMAL else None
        out[int(lab)] = e
    return out, len(kept) - 1, len(submitted), submitted

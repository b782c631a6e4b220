"""tests/near_optimal_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The definition of Solution.variability(gap=..., absolute_gap=...) (DESIGN.md section 2i) in NumPy over the C oracle:
the allowance, the bound tableau of a final tableau (rule 1), and the ranges of a list of labels with the LPs rule 3
leaves out (rules 2 to 4).  A target LP on the bound tableau is oracle/variability.target run on it: the one-edit cost
scenario with the cycle check on, exactly as section 2h runs it on the face."""
from __future__ import annotations

import numpy as np

from oracle import variability as OV

SIGN_BIT = np.uint64(1) << np.uint64(63)


def allowance(gap, absolute_gap, m00):
    """t = max(absolute_gap, gap * |z|) with z = -sigma * M[0,0]: |z| = |M[0,0]| for either sense."""
    return max(float(absolute_gap), float(gap) * abs(float(m00)))


def fresh_label(n_index, last_element_index):
    """l*: one past the parent's label space, i.e. past both its label tables and the labels cut rows took."""
    return max(int(n_index), int(last_element_index))


def bound(M, vrow, vcol, t, label):
    """(B, vrow', vcol') of the final tableau (M, vrow, vcol) for allowance t and the new label (rule 1), B at its
    logical width: rows 1..H-1 of M bit for bit, row 0 +0, B[H,0] = t and B[H,c] = -M[0,c] as a sign flip."""
    M = np.ascontiguousarray(M, dtype=np.float64)
    H, W = M.shape
    B = np.zeros((H + 1, W), dtype=np.float64)
    B[1:H] = M[1:]
    B[H, 0] = t
    B[H, 1:] = (np.ascontiguousarray(M[0, 1:]).view(np.uint64) ^ SIGN_BIT).view(np.float64)
    vrow_b = np.append(np.asarray(vrow, dtype=np.int32), np.int32(label)).astype(np.int32)
    return B, vrow_b, np.asarray(vcol, dtype=np.int32).copy()


def ranges(M, vrow, vcol, precision, labels, t, label):
    """Rules 2 to 4 for `labels` on the final tableau (M, vrow, vcol) and allowance t > 0: ({label: {"value", "min",
    "max", "argmin", "argmax"}}, free, lps, the submitted (label, sense) list in order).  argmin / argmax are (column 0,
    row labels) of the vertex of B reached, the final tableau's own where no LP runs, None where the LP gave no
    answer."""
    M = np.asarray(M, dtype=np.float64)
    B, vrow_b, vcol_b = bound(M, vrow, vcol, t, label)
    row_of = {int(vrow[r]): r for r in range(1, len(vrow))}
    here = (M[:, 0].copy(), np.asarray(vrow, dtype=np.int32).copy())
    out, submitted = {}, []
    for lab in labels:
        r = row_of.get(int(lab))
        value = float(M[r, 0]) if r is not None else 0.0
        e = {"value": value, "min": value, "max": value, "argmin": here, "argmax": here}
        for s in ([-1, 1] if r is not None else [1]):  # a non-basic label sits at its minimum, 0
            status, ev, _, _, rhs, vr = OV.target(B, vrow_b, vcol_b, precision, int(lab), s)
            submitted.append((int(lab), s))
            side = "max" if s > 0 else "min"
            e[side] = OV.end(status, ev, s)
            e["arg" + side] = (rhs, vr) if status == OV.OPTIMAL else None
        out[int(lab)] = e
    return out, M.shape[1] - 1, len(submitted), submitted

"""oracle/sensitivity.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

NumPy restatement of the sensitivity report (DESIGN.md section 2b) over a final tableau and its index maps: the
ratio-test bounds jslp_sensitivity computes on the device (`bounds`), and the whole report that
Solution.sensitivity() returns, built from the oracle's own solve (`report`).  Every quotient is the same IEEE
division of the same two operands as on the device, so the bounds compare bit for bit."""
from __future__ import annotations

import math

import numpy as np

from . import ref_model

INF = math.inf


def _unrestricted(idx, unrestricted) -> bool:
    return unrestricted is not None and 0 <= idx < len(unrestricted) and bool(unrestricted[idx])


def bounds(M, vrow, vcol, unrestricted, precision):
    """(col_lo, col_hi, row_lo, row_hi) of the final tableau M (H x W):
    col_lo[c] / col_hi[c] = max / min of -M[r,0] / M[r,c] over rows r >= 1 whose basic variable is restricted, with
    M[r,c] > P / M[r,c] < -P; row_lo[r] / row_hi[r] = max / min of M[0,c] / M[r,c] over restricted columns c >= 1
    with M[r,c] > P / M[r,c] < -P, and 0 for an unrestricted column with |M[r,c]| > P.  -0 counts as +0 and a NaN
    quotient (from non-finite entries) takes no part; an empty set gives -inf / +inf, as do row 0 and column 0."""
    M = np.asarray(M, dtype=np.float64)
    H, W = M.shape
    P = precision
    A = M[1:, :]
    pos, neg = A > P, A < -P
    live = np.arange(W) >= 1
    unres_col = np.array([c >= 1 and _unrestricted(int(vcol[c]), unrestricted) for c in range(W)], dtype=bool)
    restricted_row = np.array([not _unrestricted(int(vrow[r]), unrestricted) for r in range(1, H)], dtype=bool)[:, None]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        qc = (-A[:, :1]) / A + 0.0
        qr = M[:1, :] / A + 0.0
    take = live & restricted_row & ~np.isnan(qc)
    col_lo = np.max(np.where(pos & take, qc, -INF), axis=0, initial=-INF)
    col_hi = np.min(np.where(neg & take, qc, INF), axis=0, initial=INF)
    rc = live & ~unres_col & ~np.isnan(qr)
    hit_unres = ((pos | neg) & unres_col).any(axis=1)
    row_lo = np.max(np.where(pos & rc, qr, -INF), axis=1, initial=-INF)
    row_hi = np.min(np.where(neg & rc, qr, INF), axis=1, initial=INF)
    row_lo = np.where(hit_unres, np.maximum(row_lo, 0.0), row_lo)
    row_hi = np.where(hit_unres, np.minimum(row_hi, 0.0), row_hi)
    return col_lo, col_hi, np.concatenate([[-INF], row_lo]), np.concatenate([[INF], row_hi])


def json_row_names(jm: dict) -> list:
    """The JSON constraint name of each row loadJson builds from `constraints`, in row order (model.ts:288-323):
    `min` before `max`, two rows for `equal`."""
    names = []
    for cid in ref_model.js_keys(jm["constraints"]):
        spec = jm["constraints"][cid] if isinstance(jm["constraints"][cid], dict) else {}
        if spec.get("equal") is None:
            names += [cid] * ((spec.get("min") is not None) + (spec.get("max") is not None))
        else:
            names += [cid, cid]
    return names


def report(jm: dict, sol) -> dict:
    """The sensitivity report of `sol` = ref_model.solve_full(jm) (a continuous LP solved to optimality)."""
    model, tab = sol.model, sol.tableau
    M = tab.matrix()
    vrow, vcol = tab.maps()
    unres = np.zeros(M.shape[0] + M.shape[1] - 2, dtype=np.uint8)
    for i in model.unrestrictedVariables:
        unres[i] = 1
    col_lo, col_hi, row_lo, row_hi = bounds(M, vrow, vcol, unres, model.precision)
    sigma = -1.0 if model.isMinimization else 1.0
    row_of = {int(vrow[r]): r for r in range(1, len(vrow))}
    col_of = {int(vcol[c]): c for c in range(1, len(vcol))}
    names = json_row_names(jm)
    constraints, duals = [], {}
    for k, con in enumerate(model.constraints):
        name = names[k] if k < len(names) else con.index
        s = 1.0 if con.isUpperBound else -1.0
        if con.index in row_of:
            v = float(M[row_of[con.index], 0])
            slack, dual = v, 0.0
            rng = (con.rhs - v, INF) if s > 0 else (-INF, con.rhs + v)
        else:
            c = col_of[con.index]
            slack, dual = 0.0, -sigma * s * float(M[0, c])
            rng = (con.rhs + col_lo[c], con.rhs + col_hi[c]) if s > 0 else (con.rhs - col_hi[c], con.rhs - col_lo[c])
        constraints.append({"name": name, "type": "max" if s > 0 else "min", "rhs": con.rhs, "slack": slack,
                            "dual": dual, "range": {"min": float(rng[0]), "max": float(rng[1])}})
        duals[name] = duals.get(name, 0.0) + dual
    fixed = ref_model.presolve(model)[1] if model.usePresolve else {}
    variables = {}
    for var in model.variables:
        if var.index in row_of:
            r = row_of[var.index]
            value, reduced = float(M[r, 0]), 0.0
            rng = ((var.cost + row_lo[r], var.cost + row_hi[r]) if sigma > 0 else
                   (var.cost - row_hi[r], var.cost - row_lo[r]))
        else:
            c = col_of[var.index]
            value, reduced = 0.0, sigma * float(M[0, c])
            if var.index in model.unrestrictedVariables:
                rng = (var.cost, var.cost)
            else:
                rng = (-INF, var.cost - M[0, c]) if sigma > 0 else (var.cost + M[0, c], INF)
        is_fixed = var in fixed
        variables[var.id] = {"value": value, "cost": var.cost, "reducedCost": reduced,
                             "range": None if is_fixed else {"min": float(rng[0]), "max": float(rng[1])},
                             "fixed": is_fixed}
    return {"constraints": constraints, "duals": duals, "variables": variables}

"""oracle/parametric.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

NumPy restatement of the parametric path (DESIGN.md section 2d) from any optimal tableau: the direction, the step
bound, the shift and the other half of each pivot are computed here with the same IEEE operations as on the device,
and every pivot is done by the C oracle (ref_model.OracleTableau.pivot), rebuilt from the shifted matrix at each
breakpoint.  `path` mirrors jslp_parametric's outputs record for record, so the two compare bit for bit; `result`
shapes them as Solution.parametric() does."""
from __future__ import annotations

import math

import numpy as np

from . import ref_model

RUNNING, REACHED, INFEASIBLE, UNBOUNDED, LIMIT = 0, 1, 2, 3, 4
STOPS = {REACHED: "reached", INFEASIBLE: "infeasible", UNBOUNDED: "unbounded", LIMIT: "limit"}


def _unres(idx, unrestricted) -> bool:
    return unrestricted is not None and 0 <= idx < len(unrestricted) and bool(unrestricted[idx])


def min_quotient(num, den, unres, precision):
    """(value, position) of the smallest quotient num / den: a restricted candidate takes part when den < -P, an
    unrestricted one offers 0 when |den| > P; a quotient below 0 or -0 counts as +0, a NaN one takes no part; the
    lowest position wins ties.  (inf, -1) when nothing takes part."""
    num, den = np.asarray(num, dtype=np.float64), np.asarray(den, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        q = num / den
    q = np.where(q > 0, q, np.where(np.isnan(q), np.nan, 0.0))
    cand = np.full(len(num), math.inf)
    take = ~unres & (den < -precision)
    cand[take] = q[take]
    cand[unres & (np.abs(den) > precision)] = 0.0
    cand[np.isnan(cand)] = math.inf
    if not np.any(cand < math.inf):
        return math.inf, -1
    i = int(np.argmin(cand))
    return float(cand[i]), i


def leaving_row(M, c, is_neg, precision):
    """The reference's phase-2 ratio test on column c (simplex.ts:271-296), degenerate early exit included; -1 when
    no row bounds the step."""
    best, row = math.inf, -1
    for r in range(1, M.shape[0]):
        col, rhs = float(M[r, c]), float(M[r, 0])
        if -precision < col < precision:
            continue
        if col > 0 and precision > rhs > -precision:
            return r
        quo = (-rhs) / col if is_neg else rhs / col
        if quo > precision and best > quo:
            best, row = quo, r
    return row


def path(M, vrow, vcol, unrestricted, precision, kind, labels, signs, theta0, target, max_breaks):
    """jslp_parametric restated: {"records": [(theta, obj_raw, dobj, r, c, leaving, entering), ...], "stop": code,
    "end_rhs": column 0 at the end, "end_vrow": row labels at the end}."""
    M = np.array(M, dtype=np.float64)
    vrow = np.array(vrow, dtype=np.int32)
    vcol = np.array(vcol, dtype=np.int32)
    P = precision
    g = 1.0 if target >= theta0 else -1.0
    theta = float(theta0)
    records, stop = [], None
    while True:
        if len(records) >= max_breaks:
            stop = LIMIT
            break
        H, W = M.shape
        rho = g * (target - theta)
        row_of = {int(vrow[r]): r for r in range(1, H)}
        col_of = {int(vcol[c]): c for c in range(1, W)}
        unres_col = np.array([_unres(int(vcol[c]), unrestricted) for c in range(1, W)], dtype=bool)
        if kind == 0:
            D = None
            for lab, s in zip(labels, signs):
                if lab in col_of:
                    Dk = s * M[:, col_of[lab]]
                else:
                    Dk = np.zeros(H)
                    Dk[row_of[lab]] = s
                D = Dk if D is None else D + Dk
            restricted = np.array([not _unres(int(vrow[r]), unrestricted) for r in range(1, H)], dtype=bool)
            val, i = min_quotient(np.where(restricted, -M[1:, 0], 0.0), np.where(restricted, D[1:], 0.0),
                                  np.zeros(H - 1, dtype=bool), P)
            reach = i < 0 or val >= rho
            t = rho if reach else val
            rstar = -1 if reach else 1 + i
            nz = D != 0
            col0 = M[:, 0].copy()
            col0[nz] = M[nz, 0] + t * D[nz]
            if rstar >= 0:
                col0[rstar] = 0.0
            M[:, 0] = col0
            theta = target if reach else theta + g * t
            obj, d0 = float(M[0, 0]), float(D[0])
            if reach:
                records.append((theta, obj, d0, -1, -1, -1, -1))
                stop = REACHED
                break
            val, i = min_quotient(M[0, 1:], M[rstar, 1:], unres_col, P)
            if i < 0:
                records.append((theta, obj, d0, rstar, -1, -1, -1))
                stop = INFEASIBLE
                break
            cstar = 1 + i
        else:
            lab, sg = labels[0], signs[0]
            if lab in row_of:
                E = (-sg) * M[row_of[lab], :]
            else:
                E = np.zeros(W)
                E[col_of[lab]] = sg
            val, i = min_quotient(M[0, 1:], -E[1:], unres_col, P)
            reach = i < 0 or val >= rho
            t = rho if reach else val
            cstar = -1 if reach else 1 + i
            nz = E != 0
            row0 = M[0, :].copy()
            row0[nz] = M[0, nz] + t * E[nz]
            if cstar >= 0:
                row0[cstar] = 0.0
            M[0, :] = row0
            theta = target if reach else theta + g * t
            obj, d0 = float(M[0, 0]), float(E[0])
            if reach:
                records.append((theta, obj, d0, -1, -1, -1, -1))
                stop = REACHED
                break
            is_neg = _unres(int(vcol[cstar]), unrestricted) and E[cstar] < 0
            rstar = leaving_row(M, cstar, is_neg, P)
            if rstar < 0:
                records.append((theta, obj, d0, -1, cstar, -1, -1))
                stop = UNBOUNDED
                break
        records.append((theta, obj, d0, rstar, cstar, int(vrow[rstar]), int(vcol[cstar])))
        tab = ref_model.OracleTableau(M, vrow, vcol, precision=P, check_cycles=False)
        tab.pivot(rstar, cstar)
        M = tab.matrix()
        vrow, vcol = tab.maps()
    return {"records": records, "stop": stop, "end_rhs": M[:, 0].copy(), "end_vrow": np.array(vrow)}


def signs_for(kind, row_signs_or_sigma, theta0, target):
    """The signs jslp_parametric takes: g * s_i per moved row, or g * sigma for a cost."""
    g = 1.0 if target >= theta0 else -1.0
    return [g * s for s in row_signs_or_sigma]


def result(p, sigma, theta0, target, start_obj_raw):
    """The pieces of Solution.parametric() from a `path` output, with labels left as labels."""
    g = 1.0 if target >= theta0 else -1.0
    pieces, theta, res = [], float(theta0), -sigma * start_obj_raw
    for th, obj, d0, r, c, lv, en in p["records"]:
        pivoted = r >= 0 and c >= 0
        pieces.append({"from": theta, "to": th, "result": {"from": res, "to": -sigma * obj}, "slope": -sigma * g * d0,
                       "leaving": lv if pivoted else None, "entering": en if pivoted else None})
        theta, res = th, -sigma * obj
    return {"pieces": pieces, "stop": STOPS[p["stop"]], "end": theta, "result": res}

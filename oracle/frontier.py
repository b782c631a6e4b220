"""oracle/frontier.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

NumPy restatement of the two-objective frontier (DESIGN.md section 2g) from any optimal tableau of the first
objective: the pricing of the second objective in the contract's summation order, the weight path with the direction
carried as the optional row of the C oracle (ref_model.OracleTableau, simplex.ts:393-412), the vertex rule, and
Frontier() end to end over ref_model.solve_full.  `path` mirrors jslp_frontier's outputs record for record and point
for point, so the two compare bit for bit."""
from __future__ import annotations

import numpy as np

from . import ref_model
from .parametric import LIMIT, REACHED, UNBOUNDED, _unres, leaving_row, min_quotient

FR_ROWS = 64
STOPS = {REACHED: "reached", UNBOUNDED: "unbounded", LIMIT: "limit"}


def price(M, vrow, vcol, c2):
    """(R2, E): R2[c] = delta(c) + the block partials in block order, each partial +0 minus C2[vrow[r]] * M[r,c] over
    the block's rows in ascending order (rows with C2 == 0 skipped); E = R2 - M[0,:]."""
    M = np.asarray(M, dtype=np.float64)
    c2 = np.asarray(c2, dtype=np.float64)
    H, W = M.shape
    R = np.zeros(W)
    R[1:] = c2[np.asarray(vcol[1:], dtype=np.int64)]
    for b0 in range(1, H, FR_ROWS):
        p = np.zeros(W)
        for r in range(b0, min(b0 + FR_ROWS, H)):
            k = c2[int(vrow[r])]
            if k != 0.0:
                p = p - k * M[r, :]
        R = R + p
    return R, R - M[0, :]


def path(M, vrow, vcol, unrestricted, precision, c2, max_breaks):
    """jslp_frontier restated: {"r2", "dir", "records": [(theta, obj_raw, dobj, r, c, leaving, entering), ...],
    "stop", "points": [(column 0, row labels, records before it), ...], "end_rhs", "end_vrow"}."""
    M = np.array(M, dtype=np.float64)
    vrow = np.array(vrow, dtype=np.int32)
    vcol = np.array(vcol, dtype=np.int32)
    P = precision
    R2, E = price(M, vrow, vcol, c2)
    out = {"r2": R2.copy(), "dir": E.copy()}
    theta, target = 0.0, 1.0
    records, points, moved, stop = [], [], True, None
    while True:
        if moved:
            points.append((M[:, 0].copy(), vrow.copy(), len(records)))
            moved = False
        if len(records) >= max_breaks:
            stop = LIMIT
            break
        H, W = M.shape
        rho = target - theta
        unres_col = np.array([_unres(int(vcol[c]), unrestricted) for c in range(1, W)], dtype=bool)
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
        theta = target if reach else theta + t
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
        moved = M[rstar, 0] != 0.0
        tab = ref_model.OracleTableau(M, vrow, vcol, precision=P, opt_rc=E[None, :], check_cycles=False)
        tab.pivot(rstar, cstar)
        M = tab.matrix()
        vrow, vcol = tab.maps()
        E = tab.optional()[0].copy()
    out.update(records=records, stop=stop, points=points, end_rhs=M[:, 0].copy(), end_vrow=np.array(vrow))
    return out


def vertices(points, starts, end, stop, precision):
    """The vertex rule: distinct points in path order, each on [its start, the next one's start] (the last until
    `end`); neighbouring equal points merge; a point whose interval is no longer than the precision drops out (except
    the final point of an unbounded path) and its weights go to the next vertex kept, or to the last one at the end;
    vertices that become neighbours and are equal merge."""
    segs = []
    for k, pt in enumerate(points):
        hi = starts[k + 1] if k + 1 < len(points) else end
        if segs and segs[-1][0] == pt:
            segs[-1][2] = hi
        else:
            segs.append([pt, starts[k], hi])
    out, pending = [], None
    for k, (pt, lo, hi) in enumerate(segs):
        if hi - lo > precision or (stop == UNBOUNDED and k == len(segs) - 1):
            lo = lo if pending is None else pending
            pending = None
            if out and out[-1][0] == pt:
                out[-1][2] = hi
            else:
                out.append([pt, lo, hi])
        elif pending is None:
            pending = lo
    if pending is not None:
        if out:
            out[-1][2] = segs[-1][2]
        else:
            out.append([segs[-1][0], pending, segs[-1][2]])
    return [tuple(s) for s in out]


def _coef(jm, vid, key):
    c = jm["variables"][vid].get(key)
    return float(c) if ref_model.js_truthy(c) else 0.0


def fixed_variables(model):
    """{Variable: value} that presolve fixed in a RefModel solve_full loaded (presolve does not read the costs, so a
    second run finds the same set)."""
    return ref_model.presolve(model)[1] if model.usePresolve else {}


def cost2(model, jm, key, sense, fixed):
    """C2 by label over a RefModel: sigma2 * c2_j, 0 for slacks and for the variables presolve fixed."""
    sigma = 1.0 if sense == "max" else -1.0
    n = len(model.variables) + len(model.constraints)
    c2 = np.zeros(n)
    for v in model.variables:
        if v not in fixed:
            c2[v.index] = sigma * _coef(jm, v.id, key)
    return c2


def shape(model, jm, keys, senses, p, fixed):
    """The Frontier() result of a `path` output over the RefModel it came from."""
    theta = [r[0] for r in p["records"]]
    end = theta[-1] if theta else 0.0
    pts, starts = [], []
    for rhs, vrow, at in p["points"]:
        row_of = {int(vrow[r]): r for r in range(1, len(vrow))}
        pts.append(tuple(fixed[v] if v in fixed else (float(rhs[row_of[v.index]]) if v.index in row_of else 0.0)
                         for v in model.variables))
        starts.append(0.0 if at == 0 else theta[at - 1])
    verts = []
    for pt, lo, hi in vertices(pts, starts, end, p["stop"], model.precision):
        objs = {}
        for key in keys:
            acc = 0.0
            for v, x in zip(model.variables, pt):
                acc += _coef(jm, v.id, key) * x
            objs[key] = acc
        verts.append({"weight": {"from": lo, "to": hi}, "objectives": objs,
                      "values": {v.id: x for v, x in zip(model.variables, pt)}})
    pivots = sum(1 for r in p["records"] if r[3] >= 0 and r[4] >= 0)
    return {"feasible": True, "objectives": dict(senses), "vertices": verts, "stop": STOPS[p["stop"]], "end": end,
            "pivots": pivots}


def Frontier(jm, precision=None):
    """Frontier() over the oracle: the first objective solved by solve_full, then `path` and the vertex rule.  Returns
    (result, details) with details = {"sol", "c2", "path"} for the tests (None when infeasible); raises ValueError
    where the host does for an unbounded first objective."""
    opt = jm["optimize"]
    keys = ref_model.js_keys(opt)
    assert len(keys) == 2, keys
    senses = {k: "max" if opt[k] == "max" else "min" for k in keys}
    working = dict(jm, optimize=keys[0], opType=senses[keys[0]])
    sol = ref_model.solve_full(working, precision)
    if not sol.feasible:
        return {"feasible": False, "objectives": senses, "vertices": [], "stop": None, "end": None, "pivots": 0}, None
    if not sol.bounded:
        raise ValueError("the first objective is unbounded; list the objectives the other way round")
    model = sol.model
    M = sol.tableau.matrix()
    vrow, vcol = sol.tableau.maps()
    unres = np.zeros(M.shape[0] + M.shape[1] - 2, dtype=np.uint8)
    for i in model.unrestrictedVariables:
        unres[i] = 1
    fixed = fixed_variables(model)
    c2 = cost2(model, working, keys[1], senses[keys[1]], fixed)
    p = path(M, vrow, vcol, unres, model.precision, c2, 4 * (M.shape[0] + M.shape[1]))
    return shape(model, working, keys, senses, p, fixed), {"sol": sol, "c2": c2, "path": p, "M": M, "vrow": vrow,
                                                          "vcol": vcol, "unres": unres}

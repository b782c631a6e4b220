"""tests/repair_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The definition of Repair() (DESIGN.md section 2k) in NumPy over the C oracle: the elastic tableau of an initial
tableau with its fixed-order row 0 (rule 1), stage 1 as ref_model.OracleTableau's simplex with the cycle check on
(rule 2), stage 2 as lexicographic_oracle.child with the model's objective followed by the same simplex (rule 3), and
the whole call over ref_model.RefModel.build_tableau (no presolve), shaped as the host shapes it."""
from __future__ import annotations

import numpy as np

import lexicographic_oracle as LO
from oracle import ref_model
from oracle.sensitivity import json_row_names

SIGN_BIT = np.uint64(1) << np.uint64(63)
ELASTIC_TILE_ROWS = 32
OPTIMAL, INFEASIBLE, UNBOUNDED, CYCLED = LO.OPTIMAL, LO.INFEASIBLE, LO.UNBOUNDED, LO.CYCLED


def flip(a):
    return (np.ascontiguousarray(a, dtype=np.float64).view(np.uint64) ^ SIGN_BIT).view(np.float64)


def elastic(M, vrow, vcol, precision, rows, weights, label):
    """Rule 1: (E, vrow', vcol', crashed rows) for the uploaded tableau (M, vrow, vcol), the relaxable rows (increasing)
    with their weights, and the first new label l*; E at its logical width W + k."""
    M = np.ascontiguousarray(M, dtype=np.float64)
    H, W = M.shape
    k = len(rows)
    E = np.zeros((H, W + k), dtype=np.float64)
    E[1:, :W] = M[1:]
    vr, vc = np.asarray(vrow, dtype=np.int32).copy(), np.zeros(W + k, dtype=np.int32)
    vc[:W] = vcol
    crashed = []
    for j, r in enumerate(rows):
        E[r, W + j] = -1.0
        vc[W + j] = label + j
        if M[r, 0] < -precision:
            E[r, :W] = flip(M[r])
            vr[r] = label + j
            vc[W + j] = vrow[r]
            crashed.append(j)
    # row 0: one multiply per term, row order within tiles of ELASTIC_TILE_ROWS rows from +0, tiles in order from +0
    weight_of = {rows[j]: float(weights[j]) for j in crashed}
    total = np.zeros(W + k)
    for t0 in range(1, H, ELASTIC_TILE_ROWS):
        part = np.zeros(W + k)
        for r in range(t0, min(t0 + ELASTIC_TILE_ROWS, H)):
            if r in weight_of:
                part = part + weight_of[r] * E[r]
        total = total + part
    E[0] = total
    for j in range(k):
        if j not in crashed:
            E[0, W + j] = -float(weights[j])
    return E, vr, vc, [rows[j] for j in crashed]


def row_weights(jm, weights):
    """(rows, weights) as Repair(weights=...) chooses them: every row with weight 1, or the named constraints' rows
    with a number for all of them or {"min": a, "max": b} per side."""
    names = json_row_names(jm)
    kinds = []
    for cid in ref_model.js_keys(jm["constraints"]):
        spec = jm["constraints"][cid]
        if spec.get("equal") is None:
            kinds += [s for s in ("min", "max") if spec.get(s) is not None]
        else:
            kinds += ["min", "max"]
    if weights is None:
        return list(range(1, len(names) + 1)), [1.0] * len(names)
    chosen = {}
    for i, (name, kind) in enumerate(zip(names, kinds), start=1):
        w = weights.get(name)
        if isinstance(w, dict):
            w = w.get(kind)
        if w is not None:
            chosen[i] = float(w)
    rows = sorted(chosen)
    return rows, [chosen[r] for r in rows]


def repair(jm, weights=None, objective=True, gap=0.0, absolute_gap=0.0, precision=None):
    """Repair() over the oracle: (result, details) with details = {"M", "vrow", "vcol", "rows", "weights", "E",
    "vrow_e", "vcol_e", "crashed", "s1": (status, p1, p2, M, vrow, vcol), "T", "vrow_t", "vcol_t", "cost", "t",
    "s2": (...) or None, "e": the violation of each relaxable row at the returned plan}."""
    opt = jm.get("optimize")
    if isinstance(opt, dict):
        key = ref_model.js_keys(opt)[0]
        jm = dict(jm, optimize=key, opType="max" if opt[key] == "max" else "min")
    model = ref_model.RefModel(precision).loadJson(jm)
    P = model.precision
    M, vrow, vcol, _, _ = model.build_tableau()
    H, W = M.shape
    rows, w = row_weights(jm, weights)
    label = H + W - 2
    E, vr, vc, crashed = elastic(M, vrow, vcol, P, rows, w, label)
    det = {"M": M, "vrow": vrow, "vcol": vcol, "rows": rows, "weights": w, "E": E, "vrow_e": vr, "vcol_e": vc,
           "crashed": crashed, "s2": None}
    s1 = LO.solve(E, vr, vc, P)
    det["s1"] = s1
    status, p1, p2, Mx, vrow_f, _ = s1
    stage1 = {"kind": "violation", "optimum": None, "crashed": len(crashed), "pivots": p1 + p2, "width": W + len(rows),
              "height": H}
    out = {"feasible": True, "violation": None, "constraints": [], "values": None, "result": None, "stop": "reached",
           "stages": [stage1], "pivots": p1 + p2}
    if status == CYCLED:
        out["stop"] = "cycled"
        return out, det
    if status == INFEASIBLE:
        out["feasible"], out["stop"] = False, "infeasible"
        return out, det
    assert status == OPTIMAL, status
    vstar = float(Mx[0, 0]) + 0.0
    stage1["optimum"] = vstar
    key = jm.get("optimize") if isinstance(jm.get("optimize"), str) else None
    sigma = -1.0 if model.isMinimization else 1.0

    def plan_of(Mf, vrow_f):
        at = {int(vrow_f[r]): float(Mf[r, 0]) for r in range(1, len(vrow_f))}
        return (tuple(at.get(v.index, 0.0) for v in model.variables), [at.get(label + j, 0.0) for j in range(len(rows))])

    plan, e = plan_of(Mx, vrow_f)
    if objective:
        t = max(float(absolute_gap), float(gap) * abs(vstar))
        stage2 = {"kind": "face" if t == 0.0 else "bound", "allowance": t, "optimum": None, "pivots": 0,
                  "width": None, "height": None}
        out["stages"].append(stage2)
        cost = np.zeros(label + len(rows))
        cost[np.asarray(vcol[1:], dtype=np.int64)] = M[0, 1:]
        T, vrt, vct, _ = LO.child(Mx, s1[4], s1[5], P, cost, t, label + len(rows))
        det.update(T=T, vrow_t=vrt, vcol_t=vct, cost=cost, t=t)
        if T is None:
            stage2["optimum"] = sum_objective(model, jm, key, plan)
        else:
            s2 = LO.solve(T, vrt, vct, P)
            det["s2"] = s2
            status, p1, p2, M2, vrow2, _ = s2
            stage2.update(width=T.shape[1], height=T.shape[0], pivots=p1 + p2)
            out["pivots"] += p1 + p2
            if status == CYCLED:
                out["stop"] = "cycled"
            elif status == UNBOUNDED:
                out["stop"] = "unbounded"
            else:
                assert status == OPTIMAL, status
                stage2["optimum"] = -sigma * float(M2[0, 0]) + 0.0
                plan, e = plan_of(M2, vrow2)
    det["e"] = e
    violation = 0.0
    for wj, ej in zip(w, e):
        violation += wj * ej
    out["violation"] = violation
    names = json_row_names(jm)
    for r, wj, ej in zip(rows, w, e):
        if ej > P:
            con = model.constraints[r - 1]
            out["constraints"].append({"name": names[r - 1], "type": "max" if con.isUpperBound else "min",
                                       "rhs": con.rhs, "weight": wj, "violation": ej,
                                       "repairedRhs": con.rhs + ej if con.isUpperBound else con.rhs - ej})
    out["values"] = {v.id: x for v, x in zip(model.variables, plan)}
    out["result"] = sum_objective(model, jm, key, plan)
    return out, det


def sum_objective(model, jm, key, plan):
    """frontier.objective_sums: c_j * x_j accumulated in variable order (0 without an objective)."""
    acc = 0.0
    for v, x in zip(model.variables, plan):
        c = jm["variables"][v.id].get(key) if key is not None else None
        acc += (float(c) if ref_model.js_truthy(c) else 0.0) * x
    return acc

"""tests/lexicographic_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The definition of Lexicographic() (DESIGN.md section 2j) in NumPy over the C oracle: the starting tableau of the next
level from the optimum of the last one (rule 2: the section 2h face or the section 2i bound tableau, with the next
objective priced by oracle.frontier.price as row 0), the simplex of a level with the cycle check on (rule 3), and the
whole chain over ref_model.solve_full (rules 1, 3 and 5), shaped as the host shapes it."""
from __future__ import annotations

import numpy as np

import near_optimal_oracle as NO
from oracle import frontier as OF
from oracle import ref_model
from oracle import variability as OV

OPTIMAL, INFEASIBLE, UNBOUNDED, CYCLED = OV.OPTIMAL, OV.INFEASIBLE, OV.UNBOUNDED, OV.CYCLED


def child(M, vrow, vcol, precision, cost, t, label):
    """Rule 2: (T, vrow', vcol', kept) for the optimum (M, vrow, vcol) of a level, the next objective `cost` by label
    and the allowance t, T at its logical width; T is None when a face keeps only column 0."""
    M = np.asarray(M, dtype=np.float64)
    R = OF.price(M, vrow, vcol, cost)[0]
    if t == 0.0:
        kept, F, vcol_f = OV.face(M, vcol, precision)
        if len(kept) == 1:
            return None, None, None, kept
        F[0, :] = R[kept]
        return F, np.asarray(vrow, dtype=np.int32).copy(), vcol_f, kept
    B, vrow_b, vcol_b = NO.bound(M, vrow, vcol, t, label)
    B[0, :] = R
    return B, vrow_b, vcol_b, np.arange(M.shape[1], dtype=np.int32)


def solve(T, vrow, vcol, precision):
    """Rule 3: simplex() of a level's starting tableau with the cycle check on: (status, p1, p2, final tableau, row
    labels, column labels).  The labels are renamed to their rank for the run and named back, as in
    oracle/variability.target."""
    vrow, vcol = np.asarray(vrow, dtype=np.int32), np.asarray(vcol, dtype=np.int32)
    present = np.array(sorted([int(v) for v in vrow[1:]] + [int(v) for v in vcol[1:]]), dtype=np.int32)
    rank = {int(v): k for k, v in enumerate(present)}
    rename = lambda a: np.array([-1] + [rank[int(v)] for v in a[1:]], dtype=np.int32)  # noqa: E731
    tab = ref_model.OracleTableau(T, rename(vrow), rename(vcol), precision=precision,
                                  unrestricted=np.zeros(len(present), dtype=np.uint8), check_cycles=True,
                                  fast_cycles=True, is_min=True)
    st = tab.simplex()
    Mx, (vr, vc) = tab.matrix(), tab.maps()
    status = CYCLED if st.cyclePhase else INFEASIBLE if not st.feasible else UNBOUNDED if not st.bounded else OPTIMAL
    back = lambda a: np.array([-1] + [int(present[v]) for v in a[1:]], dtype=np.int32)  # noqa: E731
    return status, int(st.lastP1), int(st.lastP2), Mx, back(vr), back(vc)


def gaps(x, keys):
    return [float(x.get(k, 0.0)) for k in keys] if isinstance(x, dict) else [float(x)] * len(keys)


def chain(jm, gap=0.0, absolute_gap=0.0, precision=None):
    """Lexicographic() over the oracle: (result, levels) where levels[k] = {"T", "vrow", "vcol", "kept", "cost",
    "status", "p1", "p2", "M", "vrow_f", "vcol_f", "n_index"} of every level that ran an LP (level 1: T is None, and
    "fixed" = {id: value} of the variables presolve fixed)."""
    opt = jm["optimize"]
    keys = ref_model.js_keys(opt)
    senses = {k: "max" if opt[k] == "max" else "min" for k in keys}
    g, a = gaps(gap, keys), gaps(absolute_gap, keys)
    working = dict(jm, optimize=keys[0], opType=senses[keys[0]])
    sol = ref_model.solve_full(working, precision)
    model = sol.model
    out = {"feasible": bool(sol.feasible), "bounded": True, "stop": "reached", "objectives": None, "values": None,
           "levels": [], "pivots": 0}
    det = []
    if sol.tableau is None:  # presolve found the model infeasible
        out["stop"] = None
        out["levels"].append({"objective": keys[0], "sense": senses[keys[0]], "optimum": None, "allowance": None,
                              "kind": "solve", "width": None, "height": None, "pivots": 0})
        return out, det
    fixed = OF.fixed_variables(model)
    st = sol.state
    M = sol.tableau.matrix()
    vrow, vcol = sol.tableau.maps()
    status = CYCLED if st.cyclePhase else INFEASIBLE if not st.feasible else UNBOUNDED if not st.bounded else OPTIMAL
    n = M.shape[0] + M.shape[1] - 2  # n_index == nVars == lastElementIndex along the chain
    det.append({"T": None, "status": status, "p1": int(st.lastP1), "p2": int(st.lastP2), "M": M, "vrow_f": vrow,
                "vcol_f": vcol, "n_index": n, "fixed": {v.id: x for v, x in fixed.items()}})
    out["levels"].append({"objective": keys[0], "sense": senses[keys[0]], "optimum": None, "allowance": None,
                          "kind": "solve", "width": M.shape[1], "height": M.shape[0], "pivots": int(st.lastP2)})
    out["pivots"] = int(st.lastP1) + int(st.lastP2)
    if status == INFEASIBLE:
        out["feasible"], out["stop"] = False, None
        return out, det
    plan, alive = None, True
    for k, key in enumerate(keys):
        if k > 0:
            lv = {"objective": key, "sense": senses[key], "optimum": None, "allowance": None, "kind": None,
                  "width": None, "height": None, "pivots": 0}
            out["levels"].append(lv)
            if alive:
                t = out["levels"][k - 1]["allowance"]
                cost = np.zeros(n)
                c = OF.cost2(model, working, key, senses[key], fixed)
                cost[:len(c)] = c
                T, vr, vc, kept = child(M, vrow, vcol, model.precision, cost, t, NO.fresh_label(n, n))
                alive = T is not None
            if alive:
                if t > 0.0:
                    n += 1
                status, p1, p2, M, vrow, vcol = solve(T, vr, vc, model.precision)
                det.append({"T": T, "vrow": vr, "vcol": vc, "kept": kept, "cost": cost, "status": status, "p1": p1,
                            "p2": p2, "M": M, "vrow_f": vrow, "vcol_f": vcol, "n_index": n})
                lv.update(kind="face" if t == 0.0 else "bound", width=T.shape[1], height=T.shape[0], pivots=p2)
                out["pivots"] += p1 + p2
        if not alive:
            z = sum_objective(model, working, key, plan)
        else:
            if status in (CYCLED, UNBOUNDED):
                out["stop"] = "cycled" if status == CYCLED else "unbounded"
                out["bounded"] = status != UNBOUNDED
                break
            assert status == OPTIMAL, status
            z = -(1.0 if senses[key] == "max" else -1.0) * float(M[0, 0]) + 0.0
            row_of = {int(vrow[r]): r for r in range(1, len(vrow))}
            plan = tuple(fixed[v] if v in fixed else (float(M[row_of[v.index], 0]) if v.index in row_of else 0.0)
                         for v in model.variables)
        out["levels"][k]["optimum"] = z
        if k + 1 < len(keys):
            out["levels"][k]["allowance"] = max(a[k], g[k] * abs(z))
    if plan is not None:
        out["values"] = {v.id: x for v, x in zip(model.variables, plan)}
        out["objectives"] = {key: sum_objective(model, working, key, plan) for key in keys}
    return out, det


def sum_objective(model, jm, key, plan):
    """The host's objective sum: c_key,j * x_j accumulated in variable order."""
    acc = 0.0
    for v, x in zip(model.variables, plan):
        acc += OF._coef(jm, v.id, key) * x
    return acc

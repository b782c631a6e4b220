"""Sensitivity report of a solved continuous LP: what one more unit of each right-hand side is worth (dual), how far
each cost must move before its variable enters (reduced cost), and over which right-hand-side and cost values the
optimal basis stays optimal (ranges).  The reference has no counterpart; DESIGN.md section 2b defines every number.

The duals and reduced costs are the final cost row; the ratio tests behind the ranges read the whole tableau and run
on the device (jslp_sensitivity).  This module applies the signs of the objective sense and of each row."""
from __future__ import annotations

import math

INF = math.inf


def _check(solution, what: str = "sensitivity()") -> None:
    t = solution._tableau
    m = getattr(t, "model", None)
    if m is None:
        raise ValueError(f"{what} needs a solution of a Model (Solve(model, full=True) or Model.solve())")
    if m.getNumberOfIntegerVariables() > 0:
        raise ValueError(f"{what} is defined for continuous LPs only: the model has integer or binary variables")
    if any(c.relaxation is not None for c in m.constraints) or any(v.priority for v in m.variables):
        raise ValueError(f"{what} does not support soft constraints (weight / priority) or optional objectives")
    if not solution.feasible:
        raise ValueError(f"{what} needs an optimal solution: the LP is infeasible")
    if not solution.bounded:
        raise ValueError(f"{what} needs an optimal solution: the LP is unbounded")
    if t.handle is None or t._solved_version != t._version or solution._version != t._version:
        raise ValueError(f"{what} needs the tableau as the solve of this solution left it: "
                         "it has not been solved, or it was edited or solved again since")


def report(solution) -> dict:
    """{"constraints": [...], "duals": {...}, "variables": {...}} of `solution` (see Solution.sensitivity)."""
    _check(solution)
    t = solution._tableau
    m = t.model
    rhs, cost, vrow, vcol = t.final_state()
    col_lo, col_hi, row_lo, row_hi = t.sensitivity_bounds()
    sigma = -1.0 if m.isMinimization else 1.0
    row_of = {int(vrow[r]): r for r in range(1, len(vrow))}
    col_of = {int(vcol[c]): c for c in range(1, len(vcol))}

    constraints, duals = [], {}
    for con in m.constraints:
        name = con.name if con.name is not None else con.index
        upper = con.isUpperBound
        r = row_of.get(con.index)
        if r is not None:  # slack basic: the row is not binding
            slack, dual = float(rhs[r]), 0.0
            lo, hi = (con.rhs - slack, INF) if upper else (-INF, con.rhs + slack)
        else:
            c = col_of[con.index]
            s = 1.0 if upper else -1.0
            slack, dual = 0.0, -sigma * s * float(cost[c])
            lo, hi = ((con.rhs + float(col_lo[c]), con.rhs + float(col_hi[c])) if upper else
                      (con.rhs - float(col_hi[c]), con.rhs - float(col_lo[c])))
        constraints.append({"name": name, "type": "max" if upper else "min", "rhs": con.rhs, "slack": slack,
                            "dual": dual, "range": {"min": lo, "max": hi}})
        duals[name] = duals.get(name, 0.0) + dual

    fixed = m.presolveResult.fixedVariables if m.presolveResult is not None else {}
    variables = {}
    for v in m.variables:
        r = row_of.get(v.index)
        if r is not None:
            value, reduced = float(rhs[r]), 0.0
        else:
            c = col_of[v.index]
            value, reduced = 0.0, sigma * float(cost[c])
        if v in fixed:  # presolve fixed it and zeroed its cost: the LP says nothing about a cost range
            rng = None
        elif r is not None:
            lo, hi = ((v.cost + float(row_lo[r]), v.cost + float(row_hi[r])) if sigma > 0 else
                      (v.cost - float(row_hi[r]), v.cost - float(row_lo[r])))
            rng = {"min": lo, "max": hi}
        elif m.unrestrictedVariables.get(v.index):
            rng = {"min": v.cost, "max": v.cost}
        else:
            g = float(cost[c])
            rng = {"min": -INF, "max": v.cost - g} if sigma > 0 else {"min": v.cost + g, "max": INF}
        variables[v.id] = {"value": value, "cost": v.cost, "reducedCost": reduced, "range": rng, "fixed": v in fixed}
    return {"constraints": constraints, "duals": duals, "variables": variables}

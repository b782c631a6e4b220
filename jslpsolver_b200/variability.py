"""Alternative optima of a solved continuous LP: over all optimal solutions, the smallest and the largest value of every
variable and of every constraint's slack.  Solve() returns one optimal vertex; this says whether it is the only one
and, if not, how far each quantity can move at no cost to the objective.  The reference has no counterpart; DESIGN.md
section 2h is the contract.

With every reduced cost of the right sign, a feasible point is optimal exactly when every non-basic column with a
non-zero reduced cost stays at 0.  The library gathers the other columns into a face tableau on the device
(jslp_face_create) with a zero cost row; minimising and maximising one variable over it is the one-edit cost scenario
of section 2e, and all of them run as one jslp_scenario_batch on the face, each warm-started from the optimal basis.
This module resolves names, leaves out the LPs whose answer the tableau already shows, and shapes the result.

With gap= / absolute_gap= the ranges are taken over the plans whose objective is at most an allowance t worse than
the optimum (DESIGN.md section 2i): instead of the face, the device builds the optimal tableau with its objective
turned into one bound row (jslp_bound_create), bans no column, and runs the same target LPs on it."""
from __future__ import annotations

import math
import numbers

from .sensitivity import _check

WHAT = "variability()"
OPTIMAL, UNBOUNDED = 0, 2


def _gap(name: str, x, what: str = WHAT) -> float:
    """A gap= / absolute_gap= argument as a float: a finite, non-negative number."""
    if isinstance(x, bool) or not isinstance(x, numbers.Real):
        raise ValueError(f"{what}: {name}= takes a number, not {type(x).__name__}")
    x = float(x)
    if not (math.isfinite(x) and x >= 0.0):
        raise ValueError(f"{what}: {name}= must be finite and >= 0, not {x!r}")
    return x


def _end(status: int, eval_raw: float, sense: int):
    """The range end of a target LP: -s * eval_raw (a zero of either sign reads +0), s * inf when the face is unbounded
    that way, None when the LP gave no answer (a cycle, or an infeasible verdict from rounding)."""
    if status == OPTIMAL:
        return -sense * eval_raw + 0.0
    return sense * math.inf if status == UNBOUNDED else None


def _point(m, fixed, rhs, vrow) -> dict:
    """{id: value} of every structural variable at the vertex (column 0, row labels), unrounded; a variable presolve
    fixed takes its presolve value."""
    row_of = {int(vrow[r]): r for r in range(1, len(vrow))}
    return {v.id: fixed[v] if v in fixed else (float(rhs[row_of[v.index]]) if v.index in row_of else 0.0)
            for v in m.variables}


def cname(c):
    """A constraint's name in a report: its name, or its slack label for an unnamed row (a binary's `x <= 1`)."""
    return c.name if c.name is not None else c.index


def _select(m, variables, constraints, what: str = WHAT):
    """(variables, constraints) of model m that variables= / constraints= name, in model order (all of them for
    None); raises ValueError for a malformed list or an unknown name."""
    for arg, names in (("variables", variables), ("constraints", constraints)):
        if names is not None and (isinstance(names, (str, bytes, dict)) or not hasattr(names, "__iter__")):
            raise ValueError(f"{what}: {arg}= takes a list of names, not {type(names).__name__}")
    by_id = {v.id: v for v in m.variables}
    shown = list(m.variables)
    if variables is not None:
        variables = list(variables)
        for vid in variables:
            if vid not in by_id:
                raise ValueError(f"{what}: no variable named {vid!r}")
        shown = [v for v in m.variables if v.id in set(variables)]
    rows = list(m.constraints)
    if constraints is not None:
        constraints = list(constraints)
        known = {cname(c) for c in m.constraints}
        for name in constraints:
            if name not in known:
                raise ValueError(f"{what}: no constraint named {name!r}")
        rows = [c for c in m.constraints if cname(c) in set(constraints)]
    return shown, rows


def compute(solution, variables=None, constraints=None, points=False, gap=0.0, absolute_gap=0.0) -> dict:
    """Solution.variability(): see the module docstring."""
    _check(solution, WHAT)
    gap, absolute_gap = _gap("gap", gap), _gap("absolute_gap", absolute_gap)
    t = solution._tableau
    m = t.model
    if any(m.unrestrictedVariables.values()):
        raise ValueError(f"{WHAT} does not support unrestricted variables: re-solving from an optimum where one is "
                         "basic and negative starts with phase-1 pivots, which can end 'infeasible'")
    shown, rows = _select(m, variables, constraints)
    fixed = m.presolveResult.fixedVariables if m.presolveResult is not None else {}

    rhs, cost, vrow, vcol = t.final_state()
    # the allowance t = max(absolute_gap, gap * |z|), z = -sigma * M[0,0] the solved result (section 2i)
    allowance = max(absolute_gap, gap * abs(float(cost[0])))
    if math.isinf(allowance):
        raise ValueError(f"{WHAT}: the allowance gap * |result| overflows (gap={gap!r}, result={-float(cost[0])!r})")
    if allowance > 0.0:
        face, kept = t.bound(allowance), range(len(vcol))  # the bound row bans no column
    else:
        face, kept = t.face()
    kept = {int(c) for c in kept}
    row_of = {int(vrow[r]): r for r in range(1, len(vrow))}
    col_of = {int(vcol[c]): c for c in range(1, len(vcol))}
    here = _point(m, fixed, rhs, vrow) if points else None

    # every structural variable takes part (unique is a statement about all of them), then the reported rows
    labels = [v.index for v in m.variables if v not in fixed] + [c.index for c in rows]
    entry, targets = {}, []
    for lab in labels:
        if lab in entry:
            continue
        r = row_of.get(lab)
        value = float(rhs[r]) if r is not None else 0.0
        entry[lab] = {"value": value, "min": value, "max": value, "argmin": here, "argmax": here}
        if face is None:
            continue
        if r is not None:
            targets += [(lab, -1), (lab, 1)]
        elif col_of[lab] in kept:
            targets.append((lab, 1))
    if targets:
        try:
            out = face.scenario_batch([(1, lab, float(-s)) for lab, s in targets], list(range(len(targets) + 1)),
                                      check_cycles=True)
        finally:
            face.close()
        for k, (lab, s) in enumerate(targets):
            side = "max" if s > 0 else "min"
            status = int(out["status"][k])
            entry[lab][side] = _end(status, float(out["eval_raw"][k]), s)
            if points:
                entry[lab]["arg" + side] = (_point(m, fixed, out["rhs"][k], out["vrow"][k])
                                            if status == OPTIMAL else None)
    elif face is not None:
        face.close()

    def shaped(e, extra):
        d = {"value": e["value"], "min": e["min"], "max": e["max"], **extra}
        if points:
            d["argmin"], d["argmax"] = e["argmin"], e["argmax"]
        return d

    def spread(v):
        if v in fixed:
            return 0.0
        e = entry[v.index]
        return math.inf if e["min"] is None or e["max"] is None else e["max"] - e["min"]

    out_v = {}
    for v in shown:
        if v in fixed:
            e = {"value": fixed[v], "min": fixed[v], "max": fixed[v], "argmin": here, "argmax": here}
            out_v[v.id] = shaped(e, {"fixed": True})
        else:
            out_v[v.id] = shaped(entry[v.index], {"fixed": False})
    out_c = [{"name": cname(c), "type": "max" if c.isUpperBound else "min", "slack": shaped(entry[c.index], {})}
             for c in rows]
    exact = all(e["min"] is not None and e["max"] is not None for e in entry.values())
    report = {"unique": all(spread(v) <= t.precision for v in m.variables), "exact": exact, "variables": out_v,
              "constraints": out_c, "free": len(kept) - 1, "lps": len(targets)}
    if allowance > 0.0:
        report["allowance"] = allowance
    return report

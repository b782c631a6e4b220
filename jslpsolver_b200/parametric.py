"""Parametric analysis of a solved continuous LP: how the optimal result moves as one right-hand side or one cost moves
from its current value to a target, and where the optimal basis changes on the way.  It answers what lies past the
end of a sensitivity range.  The reference has no counterpart; DESIGN.md section 2d is the contract.

The path starts from the optimal tableau and runs on the device (jslp_parametric): each breakpoint is one selection
kernel and one pivot, dual simplex pivots for a right-hand side and primal simplex pivots for a cost.  Between two
breakpoints the result is linear in the moved value; its slope is the dual (right-hand side) or the variable's value
(cost), read from the tableau.  The user's tableau is left as it was.  This module resolves names, sets the direction
signs and shapes the result."""
from __future__ import annotations

import math

from .sensitivity import _check

STOPS = {1: "reached", 2: "infeasible", 3: "unbounded", 4: "limit"}


def _constraint_rows(m, name, side, what="parametric()", pick="pass side='min' or side='max'"):
    """(labels in tableau order, their row signs s_i, the side reported, the current value) of `name`.  `what` and
    `pick` word the errors for the caller (its name, and how it chooses one bound of a min+max constraint)."""
    rows = [c for c in m.constraints if (c.name if c.name is not None else c.index) == name]
    if not rows:
        raise ValueError(f"{what}: no constraint named {name!r}")
    if side not in (None, "min", "max", "equal"):
        raise ValueError(f"{what}: side must be 'min', 'max' or 'equal', not {side!r}")
    if len(rows) == 2:
        both_equal = rows[0].rhs == rows[1].rhs
        if side in ("min", "max"):
            rows = [c for c in rows if c.isUpperBound == (side == "max")]
        elif side == "equal" or both_equal:
            if not both_equal:
                raise ValueError(f"{what}: constraint {name!r} is not an equality; {pick}")
            side = "equal"
        else:
            raise ValueError(f"{what}: constraint {name!r} has a min and a max bound; {pick}")
    else:
        kind = "max" if rows[0].isUpperBound else "min"
        if side not in (None, kind):
            raise ValueError(f"{what}: constraint {name!r} has only a {kind!r} bound")
        side = kind
    return [c.index for c in rows], [1.0 if c.isUpperBound else -1.0 for c in rows], side, float(rows[0].rhs)


def _free_variable(m, variable, what="parametric()"):
    """The Variable with id `variable`; presolve must not have fixed it (that zeroes its cost, section 2b)."""
    var = next((v for v in m.variables if v.id == variable), None)
    if var is None:
        raise ValueError(f"{what}: no variable named {variable!r}")
    fixed = m.presolveResult.fixedVariables if m.presolveResult is not None else {}
    if var in fixed:
        raise ValueError(f"{what}: presolve fixed {variable!r} and zeroed its cost, so the LP has no cost to move")
    return var


def compute(solution, constraint=None, variable=None, side=None, to=None, max_breaks=None) -> dict:
    """Solution.parametric(): see the module docstring.  `max_breaks` caps the pieces (default 4 (H + W))."""
    _check(solution, "parametric()")
    if (constraint is None) == (variable is None):
        raise ValueError("parametric() takes exactly one of constraint= and variable=")
    if isinstance(to, bool) or not isinstance(to, (int, float)) or not math.isfinite(to):
        raise ValueError("parametric() needs a finite target value `to`")
    t = solution._tableau
    m = t.model
    sigma = -1.0 if m.isMinimization else 1.0
    if constraint is not None:
        labels, s, side, start = _constraint_rows(m, constraint, side)
        kind, name = 0, constraint
    else:
        if side is not None:
            raise ValueError("parametric(): side applies to constraints only")
        var = _free_variable(m, variable)
        labels, s, start = [var.index], [sigma], float(var.cost)
        kind, name = 1, variable
    target = float(to)
    g = 1.0 if target >= start else -1.0
    rhs0 = t.final_state()[0]
    cap = 4 * (t.height + t.width) if max_breaks is None else int(max_breaks)
    out = t.parametric_path(kind, labels, [g * x for x in s], start, target, cap)

    by_index = {c.index: c for c in m.constraints}
    var_of = {v.index: v for v in m.variables}

    def ref(label):
        if label < 0:
            return None
        if label in var_of:
            return {"variable": var_of[label].id}
        c = by_index[label]
        return {"constraint": c.name if c.name is not None else c.index, "type": "max" if c.isUpperBound else "min"}

    pieces = []
    theta, result = start, -sigma * float(rhs0[0])
    for k in range(len(out["theta"])):
        end, res = float(out["theta"][k]), -sigma * float(out["obj_raw"][k])
        r, c, leaving, entering = (int(x) for x in out["rc_lbl"][k])
        pivoted = r >= 0 and c >= 0
        pieces.append({"from": theta, "to": end, "result": {"from": result, "to": res},
                       "slope": -sigma * g * float(out["dobj"][k]),
                       "leaving": ref(leaving) if pivoted else None, "entering": ref(entering) if pivoted else None})
        theta, result = end, res
    row_of = {int(out["end_vrow"][r]): r for r in range(1, len(out["end_vrow"]))}
    values = {v.id: float(out["end_rhs"][row_of[v.index]]) if v.index in row_of else 0.0 for v in m.variables}
    return {"kind": "rhs" if kind == 0 else "cost", "name": name, "side": side if kind == 0 else None,
            "from": start, "to": target, "pieces": pieces, "stop": STOPS[out["stop"]], "end": theta,
            "result": result, "values": values}

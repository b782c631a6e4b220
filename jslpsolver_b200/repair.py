"""Repair of an infeasible continuous LP: the least weighted relaxation of its rows, then the model's objective
optimised over the plans that reach it.  It answers "what is the smallest change to my limits that makes this model
solvable, and what is the best plan then?", the step after iis() (the feasibility relaxation of commercial solvers).
`Repair(model, weights)` takes a JSON model; no earlier solve is needed.  The reference has no counterpart; DESIGN.md
section 2k is the contract.

Every relaxable row i gets a violation e_i >= 0 in the constraint's own units: a `max` row becomes a.x <= rhs + e_i,
a `min` row a.x >= rhs - e_i.  Stage 1 minimises V = sum_i w_i e_i.  The device builds that elastic tableau from the
model's initial tableau in one call (jslp_elastic_create), with every row that starts infeasible crashed onto its
violation, so stage 1 starts primal feasible whenever those rows may all be relaxed.  Stage 2 is one lexicographic
step (jslp_lex_next, section 2j) with the model's own objective over the plans whose violation is at most V* + t.
Presolve is not run: its fixings and removed rows rest on rows the repair may relax.  This module checks the model
and the weights, runs both stages and shapes the result."""
from __future__ import annotations

import math
import numbers
from typing import Any, Optional

from . import validation
from .frontier import _refuse, objective_sums
from .model import _truthy, object_keys
from .parametric import _constraint_rows
from .variability import _gap

WHAT = "Repair()"
PICK = "give {'min': ..., 'max': ...}"
MAX_WIDTH = 25600  # the pivot step stages a whole row in shared memory (jslp_tab_create refuses wider tableaux)


def _weight(x, what: str, caller: str = WHAT) -> float:
    if isinstance(x, bool) or not isinstance(x, numbers.Real):
        raise ValueError(f"{caller}: {what} must be a number, not {type(x).__name__}")
    x = float(x)
    if not (math.isfinite(x) and x > 0.0):
        raise ValueError(f"{caller}: {what} must be finite and > 0, not {x!r}")
    return x


def relaxable_rows(m, weights, what: str = WHAT) -> tuple:
    """(rows, weights): the tableau rows (1-based, increasing) that may be relaxed and their weights.  weights=None
    relaxes every row with weight 1; a dict {name: w} relaxes the rows of the constraints it names, `w` a number for
    every row of that constraint or {"min": a, "max": b} per side, as scenarios() reads a right-hand side."""
    row_of = {c.index: r for r, c in enumerate(m.constraints, start=1)}
    if weights is None:
        return list(range(1, len(m.constraints) + 1)), [1.0] * len(m.constraints)
    if not isinstance(weights, dict):
        raise ValueError(f"{what}: weights= takes a dict of constraint name -> weight, not {type(weights).__name__}")
    chosen = {}
    for name, value in weights.items():
        if isinstance(value, dict):
            if not value:
                raise ValueError(f"{what}: constraint {name!r}: the dict needs a 'min' and / or a 'max' key")
            for side, v in value.items():
                if side not in ("min", "max"):
                    raise ValueError(f"{what}: constraint {name!r}: side must be 'min' or 'max', not {side!r}")
                w = _weight(v, f"the {side} weight of {name!r}", what)
                for label in _constraint_rows(m, name, side, what, PICK)[0]:
                    chosen[row_of[label]] = w
        else:
            labels = [c.index for c in m.constraints if (c.name if c.name is not None else c.index) == name]
            if not labels:
                raise ValueError(f"{what}: no constraint named {name!r}")
            w = _weight(value, f"the weight of {name!r}", what)
            for label in labels:
                chosen[row_of[label]] = w
    rows = sorted(chosen)
    return rows, [chosen[r] for r in rows]


def objective_row(it, n_labels: int) -> list:
    """The model's objective by label: row 0 of the initial tableau at each structural label, 0 for slacks and for the
    violation labels."""
    cost = [0.0] * n_labels
    for c in range(1, it.matrix.shape[1]):
        cost[int(it.varIndexByCol[c])] = float(it.matrix[0, c])
    return cost


def _vertex(rhs, vrow) -> dict:
    return {int(vrow[r]): float(rhs[r]) for r in range(1, len(vrow))}


def one_objective(model: dict, what: str = WHAT) -> dict:
    """The model with a one-key `optimize` dict written as `optimize` / `opType`; several keys are refused."""
    opt = model.get("optimize")
    if isinstance(opt, dict):
        keys = object_keys(opt)
        if len(keys) > 1:
            raise ValueError(f"{what} takes one objective: `optimize` has {len(keys)}")
        if keys:
            model = dict(model, optimize=keys[0], opType="max" if opt[keys[0]] == "max" else "min")
    return model


def check_width(W: int, k: int, what: str = WHAT) -> None:
    """Refuses an elastic tableau of W + k columns beyond the pivot step's cap."""
    if W + k > MAX_WIDTH:
        raise ValueError(f"{what}: the elastic tableau needs {W + k} columns ({W} of the model and "
                         f"{k} violations), beyond the pivot step's cap of {MAX_WIDTH} columns")


def allowance(gap: float, absolute_gap: float, vstar: float, what: str = WHAT) -> float:
    """Stage 2's t = max(absolute_gap, gap * V*), refused when it overflows to infinity."""
    t = max(absolute_gap, gap * abs(vstar))
    if math.isinf(t):
        raise ValueError(f"{what}: the allowance gap * V* overflows (gap={gap!r}, V*={vstar!r})")
    return t


def report(out: dict, instance, model: dict, key, rows, w, plan, e) -> None:
    """Fills out's "violation" (sum w_j e_j in row order), "constraints" (the rows with e_j > P, their repaired
    right-hand sides), "values" and "result" from a plan and the violations e_j of the relaxable rows."""
    violation = 0.0
    for wj, ej in zip(w, e):
        violation += wj * ej
    out["violation"] = violation
    for r, wj, ej in zip(rows, w, e):
        if ej > instance.precision:
            con = instance.constraints[r - 1]
            upper = con.isUpperBound
            out["constraints"].append({"name": con.name if con.name is not None else con.index,
                                       "type": "max" if upper else "min", "rhs": con.rhs, "weight": wj,
                                       "violation": ej, "repairedRhs": con.rhs + ej if upper else con.rhs - ej})
    out["values"] = {v.id: x for v, x in zip(instance.variables, plan)}
    out["result"] = objective_sums(instance, model, [key], plan)[key]


def Repair(solver, model: Any, weights=None, *, objective: bool = True, gap=0.0, absolute_gap=0.0,
           precision: Optional[float] = None, validate: bool = False) -> dict:
    """See the module docstring.  `solver` supplies the engine settings of the tableau (Solver._instance)."""
    if validate:
        model = validation.validate(model)
    if not model:
        raise ValueError("Solver requires a model to operate on")
    if not isinstance(model, dict):
        raise ValueError(f"{WHAT} takes a JSON model")
    if model.get("external"):
        raise ValueError(f"{WHAT} does not support external solvers")
    model = one_objective(model)
    _refuse(model, WHAT)
    if any(_truthy(v) for v in (model.get("unrestricted") or {}).values()):
        raise ValueError(f"{WHAT} does not support unrestricted variables: re-solving from an optimum where one is "
                         "basic and negative starts with phase-1 pivots, which can end 'infeasible'")
    gap, absolute_gap = _gap("gap", gap, WHAT), _gap("absolute_gap", absolute_gap, WHAT)

    instance = solver._instance(model, precision)  # loadJson only: no presolve
    rows, w = relaxable_rows(instance, weights)
    it = instance.initial_tableau()
    H, W = it.matrix.shape
    check_width(W, len(rows))
    sigma = -1.0 if instance.isMinimization else 1.0
    key = model.get("optimize") if isinstance(model.get("optimize"), str) else None
    first = H + W - 2  # l*: the first violation label of a freshly uploaded tableau

    def plan_of(vertex):
        return tuple(vertex.get(v.index, 0.0) for v in instance.variables), \
            [vertex.get(first + j, 0.0) for j in range(len(rows))]

    out = {"feasible": True, "violation": None, "constraints": [], "values": None, "result": None,
           "stop": "reached", "stages": [], "pivots": 0}
    parent, E, nxt = instance.tableau, None, None
    try:
        parent.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted)
        E, crashed = parent.elastic(rows, w)
        parent.close()
        s1 = {"kind": "violation", "optimum": None, "crashed": crashed, "pivots": 0, "width": E.width,
              "height": E.height}
        out["stages"].append(s1)
        E.simplex(check_cycles=True)
        st = E.lastStatus
        s1["pivots"] = int(st.phase1_pivots) + int(st.phase2_pivots)
        out["pivots"] = s1["pivots"]
        if st.cycled:
            out["stop"] = "cycled"
            return out
        if not E.feasible:  # rows that may not be relaxed conflict on their own
            out["feasible"], out["stop"] = False, "infeasible"
            return out
        if not E.bounded:
            raise RuntimeError(f"{WHAT}: the violation, a sum of non-negative terms, came out unbounded")
        rhs, cost, vrow, _ = E.final_state()
        vstar = float(cost[0]) + 0.0
        s1["optimum"] = vstar
        plan, e = plan_of(_vertex(rhs, vrow))
        if objective:
            t = allowance(gap, absolute_gap, vstar)
            s2 = {"kind": "face" if t == 0.0 else "bound", "allowance": t, "optimum": None, "pivots": 0,
                  "width": None, "height": None}
            out["stages"].append(s2)
            nxt, _ = E.lex_next(objective_row(it, E.nVars), t)
            if nxt is None:  # the face is the stage-1 plan alone: no LP runs
                s2["optimum"] = objective_sums(instance, model, [key], plan)[key]
            else:
                s2.update(width=nxt.width, height=nxt.height)
                nxt.simplex(check_cycles=True)
                st = nxt.lastStatus
                s2["pivots"] = int(st.phase1_pivots) + int(st.phase2_pivots)
                out["pivots"] += s2["pivots"]
                if st.cycled:
                    out["stop"] = "cycled"
                elif not nxt.bounded:
                    out["stop"] = "unbounded"
                elif not nxt.feasible:
                    raise RuntimeError(f"{WHAT}: stage 2 ended infeasible from a feasible start")
                else:
                    rhs, cost, vrow, _ = nxt.final_state()
                    s2["optimum"] = -sigma * float(cost[0]) + 0.0
                    plan, e = plan_of(_vertex(rhs, vrow))
    finally:
        for tab in (nxt, E, parent):
            if tab is not None:
                tab.close()
    report(out, instance, model, key, rows, w, plan, e)
    return out

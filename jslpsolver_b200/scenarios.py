"""What-if scenarios on a solved continuous LP: re-optimise many sets of right-hand-side and cost edits in one call.
DESIGN.md section 2e is the contract.

Scenario k is by definition what the sequential Model-API path returns for it: from the solved tableau, every "rhs"
entry as Constraint.setRightHandSide applies it (an equality moves its upper row, then its lower row; a {"min", "max"}
dict moves its rows in key order), then every "cost" entry as Model.setCost applies it, then simplex() with the model's
cycle check, shaped as Solve() shapes a result.  All scenarios run on the device in one call (jslp_scenario_batch),
each warm-started from the optimal tableau.  This module validates the specs, computes the differences those methods
would pass to the tableau without changing the model, and shapes the results."""
from __future__ import annotations

import math

from .parametric import _constraint_rows, _free_variable
from .sensitivity import _check
from .tableau import EPSILON, Solution, js_round, solution_set

OPTIMAL, INFEASIBLE, UNBOUNDED, CYCLED = 0, 1, 2, 3
WHAT = "scenarios()"
PICK = "give {'min': ..., 'max': ...}"


def _number(x, what, caller=WHAT):
    if isinstance(x, bool) or not isinstance(x, (int, float)) or not math.isfinite(x):
        raise ValueError(f"{caller}: {what} must be a finite number, not {x!r}")
    return x


def _entries(spec, key, caller=WHAT):
    part = spec.get(key)
    if part is None:
        return []
    if not isinstance(part, dict):
        raise ValueError(f"{caller}: {key!r} must be a dict of name -> value, not {type(part).__name__}")
    return list(part.items())


def edits_of(m, spec, what=WHAT) -> list:
    """[(kind, index, difference), ...]: what the sequential path passes to Tableau.updateRightHandSide (kind 0, the
    constraint's slack index) and Tableau.updateCost (kind 1, the variable's index) for one scenario spec, in order.
    The model is not changed.  `what` names the caller in the errors."""
    if not isinstance(spec, dict):
        raise ValueError(f"{what}: a scenario is a dict with 'rhs' and / or 'cost', not {type(spec).__name__}")
    extra = [k for k in spec if k not in ("rhs", "cost")]
    if extra:
        raise ValueError(f"{what}: unknown scenario key(s) {extra}: a scenario has 'rhs' and 'cost'")
    by_index = {c.index: c for c in m.constraints}
    out, rhs, cost = [], {}, {}  # rhs / cost: the values the edits so far assigned (the Model API assigns them)

    def set_rhs(c, value):  # Constraint.setRightHandSide (expressions.ts:144-156)
        current = rhs.get(c, c.rhs)
        if value != current:
            difference = value - current
            if c.isUpperBound:
                difference = -difference
            rhs[c] = value
            out.append((0, c.index, float(difference)))

    for name, value in _entries(spec, "rhs", what):
        if isinstance(value, dict):
            if not value:
                raise ValueError(f"{what}: constraint {name!r}: the dict needs a 'min' and / or a 'max' key")
            for side, v in value.items():
                if side not in ("min", "max"):
                    raise ValueError(f"{what}: constraint {name!r}: side must be 'min' or 'max', not {side!r}")
                labels = _constraint_rows(m, name, side, what, PICK)[0]
                set_rhs(by_index[labels[0]], _number(v, f"the {side} of {name!r}", what))
        else:
            labels = _constraint_rows(m, name, None, what, PICK)[0]
            v = _number(value, f"the right-hand side of {name!r}", what)
            # one row, or an equality: upper row, then lower row (Equality.setRightHandSide, expressions.ts:240-245)
            for c in sorted((by_index[i] for i in labels), key=lambda c: not c.isUpperBound):
                set_rhs(c, v)
    for vid, value in _entries(spec, "cost", what):  # Model.setCost (model.ts:247-256): no skip for an unchanged cost
        var = _free_variable(m, vid, what)
        v = _number(value, f"the cost of {vid!r}", what)
        difference = v - cost.get(var, var.cost)
        if not m.isMinimization:
            difference = -difference
        cost[var] = v
        out.append((1, var.index, float(difference)))
    return out


def finish(status: int, eval_raw: float, previous: float, precision: float):
    """(feasible, evaluation, bounded) of a tableau whose simplex() ended with `status`, when its evaluation was
    `previous` before: finish_lp_flags and set_evaluation (simplex.ts:51-54,73-76,86-91,265-269,298-303;
    tableau.ts:420-430).  An infeasible or cycling run leaves the evaluation as it was."""
    if status == OPTIMAL:
        rounding = js_round(1 / precision)
        return True, js_round((EPSILON + eval_raw) * rounding) / rounding, True
    if status == UNBOUNDED:
        return True, -math.inf, False
    return False, previous, True


def compute(solution, cases) -> list:
    """Solution.scenarios(): see the module docstring."""
    _check(solution, WHAT)
    if not isinstance(cases, (list, tuple)):
        raise ValueError(f"{WHAT} takes a list of scenarios, not {type(cases).__name__}")
    t = solution._tableau
    m = t.model
    edits, offsets = [], [0]
    for spec in cases:  # every spec is checked before anything runs
        edits += edits_of(m, spec)
        offsets.append(len(edits))
    if not cases:
        return []
    out = t.scenario_batch(edits, offsets)
    from .solver import Solver
    results = []
    for k in range(len(cases)):
        feasible, evaluation, bounded = finish(int(out["status"][k]), float(out["eval_raw"][k]), t.evaluation,
                                               t.precision)
        sol = Solution(t, evaluation if m.isMinimization else -evaluation, feasible, bounded)  # Tableau.getSolution
        sol.solutionSet = solution_set(out["rhs"][k], out["vrow"][k], t.precision, t.variablesPerIndex)
        results.append(Solver._simplified(sol))
    return results

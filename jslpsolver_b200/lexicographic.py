"""Lexicographic (hierarchical) objectives of a continuous LP: optimise the objectives of `optimize` in order, each one
over the plans that give up at most an allowance on every objective before it.  `Lexicographic(model)` takes the JSON
model `MultiObjective` and `Frontier()` take; the levels are its `optimize` keys in order.  The reference has no
counterpart; DESIGN.md section 2j is the contract.

The first objective is solved as Solve() solves it.  From the optimum of level k the device builds the starting
tableau of level k+1 in one call (jslp_lex_next): the optimal face when the allowance t_k = max(absolute_gap_k,
gap_k * |z_k|) is 0, the optimum with its objective turned into one bound row when t_k > 0, and in both the next
objective priced against the optimal basis as row 0.  That tableau is primal feasible, so each later level is a phase
2 from the previous optimum.  This module checks the model and the gaps, runs the levels and shapes the result."""
from __future__ import annotations

import math
from typing import Any, Optional

from . import validation
from .frontier import _refuse, cost_row, objective_sums
from .model import _truthy, object_keys
from .variability import _gap, _point

WHAT = "Lexicographic()"


def _objectives(model: dict, what: str = WHAT):
    opt = model.get("optimize")
    keys = object_keys(opt) if isinstance(opt, dict) else []
    if len(keys) < 2:
        raise ValueError(f"{what} needs `optimize` with at least two objectives in priority order, e.g. "
                         "{\"a\": \"max\", \"b\": \"min\"}")
    return keys, {k: "max" if opt[k] == "max" else "min" for k in keys}


def _gaps(name: str, x, keys, what: str = WHAT) -> list:
    """gap= / absolute_gap= as one float per level: a number applies to every level, a dict {objective: number} to
    the objectives it names (0 for the others)."""
    if isinstance(x, dict):
        for k in x:
            if k not in keys:
                raise ValueError(f"{what}: {name}= names {k!r}, which is not an objective of `optimize`")
        return [_gap(name, x[k], what) if k in x else 0.0 for k in keys]
    return [_gap(name, x, what)] * len(keys)


def allowance(key: str, gap: float, absolute_gap: float, z: float, what: str = WHAT) -> float:
    """t_k = max(absolute_gap_k, gap_k * |z_k|), refused when it overflows to infinity."""
    t = max(absolute_gap, gap * abs(z))
    if math.isinf(t):
        raise ValueError(f"{what}: the allowance of {key!r} overflows (gap={gap!r}, optimum={z!r})")
    return t


def Lexicographic(solver, model: Any, gap=0.0, absolute_gap=0.0, precision: Optional[float] = None,
                  validate: bool = False) -> dict:
    """See the module docstring.  `solver` supplies the engine settings of the tableau (Solver._instance)."""
    if validate:
        model = validation.validate(model)
    if not model:
        raise ValueError("Solver requires a model to operate on")
    if not isinstance(model, dict):
        raise ValueError(f"{WHAT} takes a JSON model")
    if model.get("external"):
        raise NotImplementedError("external solvers (src/external) are out of scope")
    keys, senses = _objectives(model)
    _refuse(model, WHAT)
    if any(_truthy(v) for v in (model.get("unrestricted") or {}).values()):
        raise ValueError(f"{WHAT} does not support unrestricted variables: re-solving from an optimum where one is "
                         "basic and negative starts with phase-1 pivots, which can end 'infeasible'")
    gaps, absolute = _gaps("gap", gap, keys), _gaps("absolute_gap", absolute_gap, keys)

    working = dict(model, optimize=keys[0], opType=senses[keys[0]])
    instance = solver._instance(working, precision)
    solution = instance.solve()
    cur = instance.tableau
    fixed = instance.presolveResult.fixedVariables if instance.presolveResult is not None else {}
    st = cur.lastStatus
    ran = st is not None  # presolve can decide infeasibility before any LP runs
    levels = [{"objective": keys[0], "sense": senses[keys[0]], "optimum": None, "allowance": None, "kind": "solve",
               "width": cur.width if ran else None, "height": cur.height if ran else None,
               "pivots": int(st.phase2_pivots) if ran else 0}]
    total = int(st.phase1_pivots) + int(st.phase2_pivots) if ran else 0
    out = {"feasible": bool(solution.feasible), "bounded": True, "stop": "reached", "objectives": None,
           "values": None, "levels": levels, "pivots": total}
    if not solution.feasible:
        out["stop"] = None
        return out
    plan, stop = None, None
    try:
        for k, key in enumerate(keys):
            if k > 0:
                lv = {"objective": key, "sense": senses[key], "optimum": None, "allowance": None, "kind": None,
                      "width": None, "height": None, "pivots": 0}
                levels.append(lv)
                if cur is not None:
                    t = levels[k - 1]["allowance"]
                    nxt, _ = cur.lex_next(cost_row(instance, working, key, senses[key], cur.nVars), t)
                    if cur is not instance.tableau:
                        cur.close()
                    cur = nxt
                if cur is not None:
                    lv.update(kind="face" if t == 0.0 else "bound", width=cur.width, height=cur.height)
                    cur.simplex(check_cycles=True)
                    st = cur.lastStatus
                    lv["pivots"] = int(st.phase2_pivots)
                    out["pivots"] += int(st.phase1_pivots) + int(st.phase2_pivots)
            if cur is None:  # a face kept only its optimum: that plan is the only one left, and no LP runs
                z = objective_sums(instance, working, [key], plan)[key]
            else:
                if st.cycled:
                    stop = "cycled"
                elif not cur.bounded:
                    stop = "unbounded"
                elif not cur.feasible:  # every level starts primal feasible: phase 1 has nothing to do
                    raise RuntimeError(f"{WHAT}: level {k + 1} ({key!r}) ended infeasible from a feasible start")
                if stop is not None:
                    break
                rhs, cost, vrow, _ = cur.final_state()
                z = -(1.0 if senses[key] == "max" else -1.0) * float(cost[0]) + 0.0
                point = _point(instance, fixed, rhs, vrow)
                plan = tuple(point[v.id] for v in instance.variables)
            levels[k]["optimum"] = z
            if k + 1 < len(keys):
                levels[k]["allowance"] = allowance(key, gaps[k], absolute[k], z)
    finally:
        if cur is not None and cur is not instance.tableau:
            cur.close()
    if stop is not None:
        out["stop"] = stop
        out["bounded"] = stop != "unbounded"
    if plan is not None:
        out["values"] = {v.id: x for v, x in zip(instance.variables, plan)}
        out["objectives"] = objective_sums(instance, working, keys, plan)
    return out

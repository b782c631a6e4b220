"""Repair of an infeasible MIP: the least weighted relaxation of its rows over integer plans, then the model's
objective optimised over the integer plans that reach it.  It answers "what is the smallest change to my limits that
gives this model an integer plan, and what is the best such plan?", the step after Conflict().  `RepairMIP(model,
weights)` takes the JSON model Repair() takes, with `ints` or `binaries`, and returns Repair()'s shape.  The reference
has no counterpart; DESIGN.md section 2r is the contract.

Repairing the LP relaxation is not enough: `2x + 2y = 3` with x, y integer has a feasible relaxation, so Repair() of
it reports a violation of 0, while every integer plan breaks the row by at least 1.  Here the elastic tableau E of
Repair() (jslp_elastic_create, section 2k rule 1) is built over the model's tableau with its integer table, and each
stage is one exact best-first branch and bound of LexicographicMIP() (section 2q rule 2) on the device: stage 1 on E
minimises V = sum_i w_i e_i over integer plans; stage 2 runs on jslp_lex_next of E's root LP optimum with the model's
objective and the allowance t + Delta, so every integer point of it has V <= V* + t.  Presolve is not run: its
fixings and removed rows rest on rows the repair may relax."""
from __future__ import annotations

from typing import Any, Optional

from . import pool, validation
from .frontier import objective_sums
from .lexicographic_mip import delta, run_stage, signed
from .mip_variability import refuse_non_mip, refuse_unrestricted
from .repair import _vertex, allowance, check_width, objective_row, one_objective, relaxable_rows, report
from .variability import _gap

WHAT = "RepairMIP()"


def stage_entry(kind: str) -> dict:
    return {"kind": kind, "optimum": None, "pivots": 0, "width": None, "height": None, "nodes": 0, "lps": 0,
            "rounds": 0, "exact": True}


def RepairMIP(solver, model: Any, weights=None, *, objective: bool = True, gap=0.0, absolute_gap=0.0,
              max_nodes=10000, width=None, precision: Optional[float] = None, validate: bool = False) -> dict:
    """See the module docstring.  `solver` supplies the engine settings of the tableau (Solver._instance)."""
    if validate:
        model = validation.validate(model)
    if not model:
        raise ValueError("Solver requires a model to operate on")
    if not isinstance(model, dict):
        raise ValueError(f"{WHAT} takes a JSON model")
    if model.get("external"):
        raise ValueError(f"{WHAT} does not support external solvers")
    model = one_objective(model, WHAT)
    refuse_non_mip(model, WHAT, "Repair()")
    refuse_unrestricted(model, WHAT)
    gap, absolute_gap = _gap("gap", gap, WHAT), _gap("absolute_gap", absolute_gap, WHAT)
    max_nodes = pool._count("max_nodes", max_nodes, 1, WHAT)
    width = None if width is None else pool._count("width", width, 1, WHAT)

    instance = solver._instance(model, precision)  # loadJson only: no presolve
    rows, w = relaxable_rows(instance, weights, WHAT)
    it = instance.initial_tableau()
    H, W = it.matrix.shape
    check_width(W, len(rows), WHAT)
    n_ints = len(it.integerIndices)
    P = instance.precision
    sense = "min" if instance.isMinimization else "max"
    key = model.get("optimize") if isinstance(model.get("optimize"), str) else None
    first = H + W - 2  # l*: the first violation label of a freshly uploaded tableau

    out = {"feasible": True, "violation": None, "constraints": [], "values": None, "result": None,
           "stop": "reached", "stages": [], "pivots": 0}
    stages = out["stages"]
    tab, E, nxt, plan = instance.tableau, None, None, None
    try:
        tab.setModel(instance)  # with the integer indices, which E inherits
        launches0 = tab.context.launches
        E, crashed = tab.elastic(rows, w)
        tab.close()
        s1 = dict(stage_entry("violation"), crashed=crashed, width=E.width, height=E.height)
        stages.append(s1)
        found = run_stage(E, s1, P, max_nodes, width, n_ints)
        state, plan = found["state"], found["witness"]
        if state == "unbounded":
            raise RuntimeError(f"{WHAT}: the violation, a sum of non-negative terms, came out unbounded")
        if state == "cycled":
            out["stop"], plan = "cycled", None
        elif state == "limit":
            if plan is None:
                raise ValueError(f"{WHAT}: the search of stage 1 hit max_nodes={max_nodes} before any integer plan; "
                                 "raise max_nodes")
            s1["exact"], s1["bound"] = False, signed("min", found["bound"])
            out["stop"] = "limit"
        elif plan is None:  # no integer plan: the rows that may not be relaxed conflict with integrality
            out["feasible"], out["stop"] = False, "infeasible"
        if plan is not None:
            vstar = s1["optimum"] = signed("min", float(plan.rhs[0]))
        if plan is not None and objective and state == "exact":
            t = allowance(gap, absolute_gap, vstar, WHAT)
            d = delta(E, s1, plan, f"{WHAT}: the root LP of stage 1")
            if d is None:
                out["stop"] = "cycled"
            else:
                s2 = dict(stage_entry("face" if t + d == 0.0 else "bound"), allowance=t)
                stages.append(s2)
                nxt, _ = E.lex_next(objective_row(it, E.nVars), t + d)
                if nxt is None:  # the face is the stage-1 plan alone: no search runs
                    s2["optimum"] = objective_sums(instance, model, [key], plan_of(instance, plan)[0])[key]
                else:
                    s2.update(width=nxt.width, height=nxt.height)
                    found = run_stage(nxt, s2, P, max_nodes, width, n_ints)
                    state, best = found["state"], found["witness"]
                    if state in ("unbounded", "cycled"):
                        out["stop"] = state
                    else:
                        if best is None and state == "exact":
                            raise RuntimeError(f"{WHAT}: stage 2 has no integer plan, but the plan of stage 1 is one")
                        if state == "limit":
                            s2["exact"], s2["bound"] = False, signed(sense, found["bound"])
                            out["stop"] = "limit"
                        if best is not None:
                            plan = best
                            s2["optimum"] = signed(sense, float(best.rhs[0]))
                        else:
                            s2["optimum"] = objective_sums(instance, model, [key], plan_of(instance, plan)[0])[key]
        out["launches"] = tab.context.launches - launches0
    finally:
        for derived in (nxt, E, tab):
            if derived is not None:
                derived.close()
    if plan is not None:
        x, at = plan_of(instance, plan)
        report(out, instance, model, key, rows, w, x, [at.get(first + j, 0.0) for j in range(len(rows))])
    for name in ("nodes", "lps", "rounds", "pivots"):
        out[name] = sum(s[name] for s in stages)
    return out


def plan_of(instance, node) -> tuple:
    """(values of the structural variables in model order, {label: value}) at an integral node's final column 0."""
    at = _vertex(node.rhs, node.vrow)
    return tuple(at.get(v.index, 0.0) for v in instance.variables), at

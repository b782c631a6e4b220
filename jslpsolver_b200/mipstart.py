"""MIP starts: seed branch and cut with known integer plans.  DESIGN.md section 2t is the contract.

Solve(model, start=plan_or_list, start_nodes=1000) / Model.solve(start=...) turns each plan ({variable: value}, a
Solve() result passed back as it is included) into a list of branching cuts on the integer columns of the tableau
Solve() branches on, runs jslp_branch_and_cut_start, and reports every start's fate under Solution.mipStart.  This
module checks the model and the plans, maps names to cut lists (`cut_lists`, no GPU needed) and builds the report."""
from __future__ import annotations

import math
import numbers

WHAT = "Solve(start=...)"
HEAD_KEYS = ("feasible", "result", "bounded", "isIntegral")  # the head of a simplified Solve() result
STATUS = ("seed", "feasible", "infeasible", "incomplete", "skipped")  # jslp_start_status.status


def check_json(model: dict, basis) -> None:
    """The refusals of a start that depend on the JSON model and the call's other arguments."""
    if basis is not None:
        raise ValueError(f"{WHAT} cannot be combined with basis=: a basis warm-starts a continuous LP")
    opt = model.get("optimize")
    if isinstance(opt, dict) and len(opt) > 1:
        raise ValueError(f"{WHAT} does not support multi-objective models (optimize with several objectives)")
    if model.get("external"):
        raise ValueError(f"{WHAT} does not support external solvers")


def check_model(m, start_nodes) -> None:
    """The refusals of a start that depend on the model alone."""
    if m.getNumberOfIntegerVariables() == 0:
        raise ValueError(f"{WHAT} is defined for MIPs only: a continuous model is warm-started with basis=")
    if any(c.relaxation is not None for c in m.constraints) or any(v.priority for v in m.variables):
        raise ValueError(f"{WHAT} does not support soft constraints (weight / priority) or optional objectives")
    if getattr(m, "branchAndCutOptions", None) or m.branchAndCutService is not None:
        raise ValueError(f"{WHAT} needs the default branch-and-cut service (no nodeSelection, branching or "
                         "useIncremental)")
    if m.tableau.distributed:
        raise ValueError(f"{WHAT} runs on one GPU: distributed branch and cut is not supported")
    if isinstance(start_nodes, bool) or not isinstance(start_nodes, numbers.Integral) or start_nodes < 1:
        raise ValueError(f"{WHAT}: start_nodes must be an integer of at least 1")


def plans(start) -> list:
    """The plans of `start`: one dict, or a list of them."""
    out = [start] if isinstance(start, dict) else start
    if not isinstance(out, (list, tuple)) or not all(isinstance(p, dict) for p in out):
        raise ValueError(f"{WHAT}: a start is a {{variable: value}} dict (a Solve() result), or a list of them")
    return list(out)


def cut_lists(m, plan_list) -> list:
    """One entry per plan: {"cuts": [(type, varIndex, value)] or None when the start is fractional, "unknown": [...],
    "ignored": [...]}.  Integer variables in integerVariables order, each fixed one giving {min, j, v} when v > 0 and
    then {max, j, v}; a missing integer variable is 0, None leaves it free, presolve-fixed ones are left to presolve."""
    by_id = {v.id: v for v in m.variables}
    fixed = set(m.presolveResult.fixedVariables) if m.presolveResult is not None else set()
    out = []
    for plan in plan_list:
        unknown, ignored, values, fractional = [], [], {}, False
        for name, value in plan.items():
            var = by_id.get(name)
            if var is None:
                if name not in HEAD_KEYS:
                    unknown.append(name)
                continue
            if not var.isInteger or var in fixed:
                ignored.append(name)
                continue
            if value is not None and (isinstance(value, bool) or not isinstance(value, numbers.Real)
                                      or not math.isfinite(value)):
                raise ValueError(f"{WHAT}: the value of {name!r} must be a finite number or None, not {value!r}")
            values[var.index] = value
        cuts = []
        for var in m.integerVariables:
            if var in fixed:
                continue
            v = values.get(var.index, 0)
            if v is None:
                continue
            r = float(math.floor(v + 0.5))
            if abs(v - r) > m.precision:
                fractional = True
                break
            if r > 0:
                cuts.append((0, var.index, r))
            cuts.append((1, var.index, r))
        out.append({"cuts": None if fractional else cuts, "unknown": unknown, "ignored": ignored})
    return out


def report(m, mapped, native, final_evaluation) -> dict:
    """Solution.mipStart: the mapped starts (cut_lists) with the native status rows of those that ran, in order, and
    the final Tableau.evaluation (minimisation sense) of the run."""
    sign = 1.0 if m.isMinimization else -1.0
    starts, seed, it = [], None, iter(native)
    for i, s in enumerate(mapped):
        row = {"status": "fractional", "result": None, "nodes": 0, "pivots": 0}
        if s["cuts"] is not None:
            st = next(it, None)
            if st is None:  # presolve proved the model infeasible: nothing ran
                row["status"] = "skipped"
            else:
                row = {"status": STATUS[st.status], "result": None if math.isnan(st.evaluation)
                       else sign * st.evaluation + 0.0, "nodes": int(st.nodes), "pivots": int(st.pivots)}
                if row["status"] == "seed":
                    seed = i
        row["unknown"], row["ignored"] = s["unknown"], s["ignored"]
        starts.append(row)
    improved = seed is not None and final_evaluation < sign * starts[seed]["result"]
    return {"starts": starts, "seed": seed, "improved": bool(improved),
            "nodes": sum(s["nodes"] for s in starts), "pivots": sum(s["pivots"] for s in starts)}


def solve(m, start, start_nodes: int = 1000):
    """Model.solve(start=...): presolve and upload as Model.solve() does, branch and cut seeded with the starts."""
    check_model(m, start_nodes)
    plan_list = plans(start)
    from .model import presolve
    if m.usePresolve and m.presolveResult is None:  # Model.solve (model.ts:427-449)
        m.presolveResult = presolve(m)
        if m.presolveResult.isInfeasible:
            m.tableau.model = m
            m.tableau.feasible = False
            sol = m.tableau.getSolution()
            sol.mipStart = report(m, cut_lists(m, plan_list), [], math.inf)
            return sol
        for variable, value in m.presolveResult.fixedVariables.items():
            variable.value = value
            variable.cost = 0
    mapped = cut_lists(m, plan_list)
    t = m.tableau
    if not m.tableauInitialized:
        t.setModel(m)
        m.tableauInitialized = True
    t.lastStartStatus = []
    sol = t.solve(start=[s["cuts"] for s in mapped if s["cuts"] is not None], start_nodes=int(start_nodes))
    sol.mipStart = report(m, mapped, t.lastStartStatus, t.evaluation)
    return sol

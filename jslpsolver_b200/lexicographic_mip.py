"""Lexicographic (hierarchical) objectives of a MIP: optimise the objectives of `optimize` in priority order, each one
over the integer plans that give up at most an allowance on every objective before it ("cheapest schedule first, then
the fewest overtime shifts among those").  `LexicographicMIP(model)` takes the JSON model `Lexicographic()` takes, with
`ints` or `binaries`, and returns the same shape.  The reference has no counterpart; DESIGN.md section 2q is the
contract.

Each level is one exact best-first branch and bound on its own tableau T_k, its node LPs batched on the device
(jslp_pool_batch with cut rows only).  T_1 is the model's initial tableau.  From the root LP optimum R_k of T_k the
device builds T_{k+1} in one call (jslp_lex_next): objective k turned into one bound row with allowance t_k + Delta_k,
where t_k = max(absolute_gap_k, gap_k * |z_k|) and Delta_k is what the level's MIP optimum loses against R_k, or the
optimal face when that sum is 0; row 0 is objective k+1 priced against R_k.  Every integer point of T_{k+1} is then
within t_k of z_k on objective k and keeps every earlier bound.  The model is loaded as Pool() loads it (no presolve,
no tolerance / timeout), so the answer is exact for the model as written, up to the node limit."""
from __future__ import annotations

import math
from typing import Any, Optional

from . import iis, pool, validation
from .frontier import cost_row, objective_sums
from .lexicographic import _gaps, _objectives, allowance
from .mip_variability import OPTIMAL, node_of, plan_values, refuse_non_mip, refuse_unrestricted, run

WHAT = "LexicographicMIP()"
OWN = (None, -1, False)  # the one target of a level's search: the node LP's own objective, minimised


def search(evaluate, P: float, max_nodes: int, width: Optional[int], wave: int) -> dict:
    """Rule 2: one level's best-first branch and bound, mip_variability.run with the single target OWN and no
    incumbent.  evaluate([(0, cuts), ...]) -> [Node, ...] are the node LPs of the level's tableau plus the cut rows.
    The first integral node to reach the top of the heap ends the search ("exact", its witness); "exact" without a
    witness means the level has no integer plan.  At "limit" the witness is the best integral node evaluated so far
    (lowest evaluation, the first one on ties), or None when none was."""
    seen: list = []

    def tracked(specs):
        nodes = evaluate(specs)
        for node in nodes:
            if node.status == OPTIMAL and node.integral and (not seen or node.evaluation < seen[0].evaluation):
                seen[:] = [node]
        return nodes

    out = run(tracked, [OWN], [math.inf], P, max_nodes, width, wave)
    state, witness = out["state"][0], out["witness"][0]
    if state == "limit":
        witness = seen[0] if seen else None
    return {"state": state, "witness": witness, "bound": out["bound"][0], "nodes": out["nodes"], "lps": out["lps"],
            "rounds": out["rounds"]}


def run_stage(cur, entry: dict, P: float, max_nodes: int, width: Optional[int], n_ints: int) -> dict:
    """Rule 2 on the tableau cur: its snapshot saved, then search() with every node LP one jslp_pool_batch region (no
    fixings, the node's cut rows, cycle check on) and the default width one wave of cur plus an 8-level dive.  The
    node LPs' pivots and the search's nodes, LPs and rounds go into entry."""
    def evaluate(specs):
        res = cur.pool_batch([([], cuts) for _, cuts in specs], check_cycles=True)
        entry["pivots"] += int(res["pivots"].sum())
        return [node_of(res, i, cur.height, cuts) for i, (_, cuts) in enumerate(specs)]

    cur.save()
    found = search(evaluate, P, max_nodes, width, iis.wave_width(cur.context, cur.height + min(n_ints, 8), cur.width))
    entry.update(nodes=found["nodes"], lps=found["lps"], rounds=found["rounds"])
    return found


def delta(cur, entry: dict, best, what: str) -> Optional[float]:
    """Rule 1's R_k and Delta_k: cur restored and its root LP solved (cycle check on), its pivots added to entry;
    Delta_k = max(0, raw M[0,0] of the optimal node best - raw M[0,0] of R_k), or None when the root LP cycled.
    `what` names the root LP in the RuntimeError raised when it has no optimum."""
    cur.restore()
    cur.simplex(check_cycles=True)
    st = cur.lastStatus
    entry["pivots"] += int(st.phase1_pivots) + int(st.phase2_pivots)
    if st.cycled:
        return None
    if not (cur.feasible and cur.bounded):
        raise RuntimeError(f"{what} has no optimum, but its search found one")
    return max(0.0, float(best.rhs[0]) - float(cur.final_state()[1][0]))


def signed(sense: str, raw: float) -> float:
    """The objective value of a raw M[0,0] (the tableau minimises, so a max objective's row holds -value)."""
    return (-raw if sense == "max" else raw) + 0.0


def level_entry(key: str, sense: str) -> dict:
    return {"objective": key, "sense": sense, "optimum": None, "allowance": None, "kind": None, "width": None,
            "height": None, "nodes": 0, "lps": 0, "rounds": 0, "pivots": 0, "exact": True}


def LexicographicMIP(solver, model: Any, gap=0.0, absolute_gap=0.0, max_nodes=10000, width=None,
                     precision: Optional[float] = None, validate: bool = False) -> dict:
    """See the module docstring.  `solver` supplies the engine settings of the tableau (Solver._instance)."""
    if validate:
        model = validation.validate(model)
    if not model:
        raise ValueError("Solver requires a model to operate on")
    if not isinstance(model, dict):
        raise ValueError(f"{WHAT} takes a JSON model")
    if model.get("external"):
        raise NotImplementedError("external solvers (src/external) are out of scope")
    keys, senses = _objectives(model, WHAT)
    refuse_non_mip(model, WHAT, "Lexicographic()")
    refuse_unrestricted(model, WHAT)
    gaps, absolute = _gaps("gap", gap, keys, WHAT), _gaps("absolute_gap", absolute_gap, keys, WHAT)
    max_nodes = pool._count("max_nodes", max_nodes, 1, WHAT)
    width = None if width is None else pool._count("width", width, 1, WHAT)

    working = dict(model, optimize=keys[0], opType=senses[keys[0]])
    instance = solver._instance(working, precision)  # loadJson only: no presolve
    tab = instance.tableau
    try:
        tab.setModel(instance)
        out = chain(tab, instance, working, keys, senses, gaps, absolute, max_nodes, width, WHAT)
    finally:
        tab.close()
    return out


def chain(tab, instance, working: dict, keys, senses: dict, gaps, absolute, max_nodes: int, width: Optional[int],
          what: str) -> dict:
    """The levels of rules 1 and 2 over keys in order, from the initial tableau tab of `instance` (loaded from
    `working`, whose objective is keys[0]; setModel done, no presolve), with allowances from gaps / absolute (one per
    key).  Returns LexicographicMIP()'s result; every tableau derived from tab is closed, tab is not.
    `what` names the caller in the refusal of a level-1 search that hits max_nodes before any integer plan."""
    n_ints = len(instance.initial_tableau().integerIndices)
    P = instance.precision
    levels: list = []
    out = {"feasible": True, "bounded": True, "stop": "reached", "objectives": None, "values": None,
           "levels": levels}
    plan, cur, arg = None, tab, 0.0
    launches0 = tab.context.launches
    try:
        for k, key in enumerate(keys):
            lv = level_entry(key, senses[key])
            levels.append(lv)
            if k > 0 and cur is not None:  # rule 1: T_k from R_{k-1}
                nxt, _ = cur.lex_next(cost_row(instance, working, key, senses[key], cur.nVars), arg)
                if cur is not tab:
                    cur.close()
                cur = nxt
            if cur is None:  # a face kept only the last plan: it is the only one left, and no search runs
                lv["optimum"] = objective_sums(instance, working, [key], plan)[key]
            else:
                lv.update(kind="initial" if k == 0 else "face" if arg == 0.0 else "bound", width=cur.width,
                          height=cur.height)
                found = run_stage(cur, lv, P, max_nodes, width, n_ints)
                state, best = found["state"], found["witness"]
                if state in ("unbounded", "cycled"):
                    out["stop"] = state
                    break
                if state == "limit":
                    if best is None and plan is None:
                        raise ValueError(f"{what}: the search of level 1 ({key!r}) hit max_nodes={max_nodes} before "
                                         "any integer plan; raise max_nodes")
                    lv["exact"], lv["bound"] = False, signed(senses[key], found["bound"])
                if best is None and state == "exact":
                    if k == 0:  # no integer plan: Conflict() explains why
                        out["feasible"], out["stop"] = False, None
                        break
                    raise RuntimeError(f"{what}: level {k + 1} ({key!r}) has no integer plan, but the plan of level "
                                       f"{k} is one")
                if best is not None:
                    at = plan_values(best.rhs, best.vrow)
                    plan = tuple(at.get(v.index, 0.0) for v in instance.variables)
                    lv["optimum"] = signed(senses[key], float(best.rhs[0]))
                else:
                    lv["optimum"] = objective_sums(instance, working, [key], plan)[key]
                if state == "limit":
                    out["stop"] = "limit"
                    break
            if k + 1 < len(keys):
                lv["allowance"] = t = allowance(key, gaps[k], absolute[k], lv["optimum"], what)
                if cur is not None:  # R_k and Delta_k
                    d = delta(cur, lv, best, f"{what}: the root LP of level {k + 1} ({key!r})")
                    if d is None:
                        out["stop"] = "cycled"
                        break
                    arg = t + d
        out["launches"] = tab.context.launches - launches0
    finally:
        if cur is not None and cur is not tab:
            cur.close()
    if out["stop"] == "unbounded":
        out["bounded"] = False
    if plan is not None:
        out["values"] = {v.id: x for v, x in zip(instance.variables, plan)}
        out["objectives"] = objective_sums(instance, working, keys, plan)
    for name in ("nodes", "lps", "rounds", "pivots"):
        out[name] = sum(lv[name] for lv in levels)
    return out

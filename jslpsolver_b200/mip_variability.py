"""Near-optimal variability of a MIP: over all integer plans whose objective is at most an allowance t worse than the
MIP optimum, the smallest and the largest value of every variable and of every constraint's slack.  It answers "which
decisions are forced, and how far can each one move if I give up a little?" for models with `ints` / `binaries`, the
question Solution.variability(gap=...) answers for continuous LPs; `Variability(model, gap=...)` takes a JSON model and
returns the same shape.  The reference has no counterpart; DESIGN.md section 2o is the contract.

The optimum z* and an optimal plan x* come from the solution-pool search with k = 1 (pool.run, no presolve).  The
root LP optimum is then turned into one bound tableau B (jslp_bound_create) whose feasible points are exactly the plans
at most t worse than z*.  Every target (a label and a sense) is an exact best-first branch and bound on B with row 0
set to +-1 on its label.  All the searches run side by side: each round takes the children of the first `width` open
nodes of every live search into one jslp_target_batch call, and the searches then commit in target order, sharing every
integral plan they meet as an incumbent of every target it improves.  `width` changes the work counters and which
witness is reported, never an exact end.  Not applied: presolve, the enhanced or incremental services' branching rules and
options.tolerance / timeout; the answer describes the model as written, and is exact up to the node limit."""
from __future__ import annotations

import heapq
import math
from typing import Any, Optional

from . import iis, pool, validation
from .model import _truthy, object_keys
from .variability import _gap, _select, cname

WHAT = "Variability()"
OPTIMAL, INFEASIBLE, UNBOUNDED, CYCLED = pool.OPTIMAL, pool.INFEASIBLE, pool.UNBOUNDED, pool.CYCLED


def _refuse(model: dict) -> None:
    if not isinstance(model, dict):
        raise ValueError(f"{WHAT} takes a JSON model")
    if model.get("external"):
        raise ValueError(f"{WHAT} does not support external solvers: solve the model with its own solver")
    refuse_non_mip(model, WHAT, "Solve(model, full=True).variability()")
    opt = model.get("optimize")
    if isinstance(opt, dict) and len(object_keys(opt)) > 1:
        raise ValueError(f"{WHAT} takes one objective: `optimize` has {len(object_keys(opt))}; use Lexicographic() "
                         "or Solve() for several")
    refuse_unrestricted(model, WHAT)


def refuse_non_mip(model: dict, what: str, continuous: str) -> None:
    """The refusals of the MIP analyses that search on a bound tableau: a model without integer or binary variables
    (`continuous` names what answers it for a continuous LP) and soft constraints."""
    if not (any(_truthy(v) for v in (model.get("ints") or {}).values()) or
            any(_truthy(v) for v in (model.get("binaries") or {}).values())):
        raise ValueError(f"{what} needs integer or binary variables: for a continuous LP use {continuous}")
    for spec in (model.get("constraints") or {}).values():
        if isinstance(spec, dict) and (spec.get("weight") is not None or spec.get("priority") is not None):
            raise ValueError(f"{what} does not support soft constraints (weight / priority): make them hard rows")


def refuse_unrestricted(model: dict, what: str) -> None:
    if any(_truthy(v) for v in (model.get("unrestricted") or {}).values()):
        raise ValueError(f"{what} does not support unrestricted variables: re-solving from an optimum where one is "
                         "basic and negative starts with phase-1 pivots; split each into two restricted variables")


class Node:
    """One node of a target search: its cut rows and its LP's verdict."""
    __slots__ = ("cuts", "status", "evaluation", "integral", "branch_var", "branch_value", "rhs", "vrow", "children")

    def __init__(self, cuts, status, evaluation, integral, branch_var, branch_value, rhs=None, vrow=None):
        self.cuts, self.status, self.evaluation = cuts, int(status), float(evaluation)
        self.integral, self.branch_var, self.branch_value = bool(integral), int(branch_var), float(branch_value)
        self.rhs, self.vrow = rhs, vrow
        self.children: Optional[list] = None


def plan_values(rhs, vrow) -> dict:
    """{label: value} of the basic labels of a node's final column 0 (rows >= 1); a label not in it is at 0."""
    return {int(vrow[r]): float(rhs[r]) for r in range(1, len(vrow))}


class _Search:
    """The best-first search of one target (label, sense s: -1 min, +1 max) on the bound tableau: it minimises the
    evaluation -s * label, lowest first and most recently pushed first on ties (pool.run's heap)."""
    __slots__ = ("k", "label", "s", "integer", "heap", "seq", "nodes", "state", "bound")

    def __init__(self, k: int, label: int, s: int, integer: bool):
        self.k, self.label, self.s, self.integer = k, label, s, integer
        self.heap, self.seq, self.nodes = [], 0, 1
        self.state = "live"  # then "exact", "limit", "unbounded" or "cycled"
        self.bound = None

    def push(self, node: Node) -> None:
        heapq.heappush(self.heap, (node.evaluation, -self.seq, node))
        self.seq += 1

    def end_bound(self, node: Node, P: float) -> float:
        """The best value of the label under node: -s * evaluation, on the integer grid for an integer label."""
        b = -self.s * node.evaluation
        if self.integer:
            b = float(math.floor(b + P)) if self.s > 0 else float(math.ceil(b - P))
        return b


def run(evaluate, targets, start: list, P: float, max_nodes: int, width: Optional[int], wave: int = 1,
        shared: bool = True) -> dict:
    """The concurrent target searches of DESIGN.md section 2o (rules 4 to 8).  targets = [(label, sense, integer)];
    a label of None stands for the node LP's own objective, so its value at an integral node is the node's evaluation
    and its sense is -1 (the lexicographic levels of section 2q).  start[k] = target k's incumbent value at x*; a
    target without one starts at -s * math.inf (math.inf for a min target, such as the label-None target).
    evaluate([(k, cuts), ...]) -> [Node, ...], the nodes' LPs on the bound tableau with row 0 set to -s_k on label_k.
    Each round evaluates the children of the first `width` open nodes (None: wave // live searches, at least 1) of
    every live search in one call, then commits the searches in target order.  With shared=False an integral plan is
    an incumbent of its own search only (the searches of section 2s run on different feasible regions).  Returns
    {"best", "witness" (Node or None: x*), "state", "bound", "nodes", "lps", "rounds"}."""
    n = len(targets)
    searches = [_Search(k, lab, s, integer) for k, (lab, s, integer) in enumerate(targets)]
    best, witness = list(start), [None] * n

    def beats(sr: _Search, value: float) -> bool:
        return sr.s * (value - best[sr.k]) > P

    def share(node: Node, owner: _Search) -> None:
        at = plan_values(node.rhs, node.vrow)
        for sr in searches if shared else [owner]:
            v = node.evaluation if sr.label is None else at.get(sr.label, 0.0)
            if beats(sr, v):
                best[sr.k], witness[sr.k] = v, node

    def commit(sr: _Search) -> None:
        """Pops in heap order until the top is not worth expanding or has no evaluated children."""
        while sr.state == "live":
            if not sr.heap or not beats(sr, sr.end_bound(sr.heap[0][2], P)):
                sr.state = "exact"
                return
            top = sr.heap[0][2]
            if not top.integral and sr.nodes >= max_nodes:
                sr.state, sr.bound = "limit", sr.end_bound(top, P)
                return
            if not top.integral and top.children is None:
                return
            heapq.heappop(sr.heap)
            if top.integral:
                share(top, sr)
                continue
            sr.nodes += len(top.children)
            for c in top.children:
                if c.status in (UNBOUNDED, CYCLED):
                    sr.state = "unbounded" if c.status == UNBOUNDED else "cycled"
                    return
            for c in top.children:
                if c.status == OPTIMAL:
                    sr.push(c)

    def settle(sr: _Search, node: Node) -> None:
        if node.status in (UNBOUNDED, CYCLED):
            sr.state = "unbounded" if node.status == UNBOUNDED else "cycled"
        elif node.status == OPTIMAL:
            sr.push(node)

    for sr, node in zip(searches, evaluate([(k, []) for k in range(n)])):
        settle(sr, node)
    count = {"lps": n, "rounds": 1}
    while True:
        for sr in searches:
            commit(sr)
        live = [sr for sr in searches if sr.state == "live"]
        if not live:
            break
        w = width if width is not None else max(1, wave // len(live))
        specs, owners = [], []
        for sr in live:
            for e in heapq.nsmallest(w, sr.heap):
                node = e[2]
                if node.integral or node.children is not None or not beats(sr, sr.end_bound(node, P)):
                    continue
                kids = pool_children(node)
                specs += [(sr.k, c) for c in kids]
                owners.append((node, len(kids)))
        done = evaluate(specs)
        count["lps"] += len(specs)
        count["rounds"] += 1
        pos = 0
        for node, m in owners:
            node.children = done[pos:pos + m]
            pos += m
    return {"best": best, "witness": witness, "state": [sr.state for sr in searches],
            "bound": [sr.bound for sr in searches], "nodes": sum(sr.nodes for sr in searches), **count}


def pool_children(node: Node) -> list:
    """The cut lists of a fractional node's children in push order: the `min ceil(x)` child, then the `max floor(x)`
    child, each replacing the same-type cut on the branching variable (branch-and-cut.ts:155-190)."""
    v, x = node.branch_var, node.branch_value
    return [pool.replace_cut(node.cuts, (0, v, float(math.ceil(x)))),
            pool.replace_cut(node.cuts, (1, v, float(math.floor(x))))]


def targets_of(shown, rows, ints: set) -> list:
    """Rule 3: (label, sense, integer) of every reported variable in model order, then every reported row, min before
    max."""
    labels = [(v.index, v.index in ints) for v in shown] + [(c.index, False) for c in rows]
    return [(lab, s, integer) for lab, integer in labels for s in (-1, 1)]


def allowance(gap: float, absolute_gap: float, opt_raw: float) -> float:
    """t = max(absolute_gap, gap * |z*|), |z*| = |M[0,0]| of the optimal plan's region."""
    t = max(absolute_gap, gap * abs(opt_raw))
    if math.isinf(t):
        raise ValueError(f"{WHAT}: the allowance gap * |optimum| overflows (gap={gap!r}, optimum={opt_raw!r})")
    return t


def optimum(found: dict, max_nodes: int):
    """Rule 1's verdict: the optimal Region of pool.run(k=1), or the refusal."""
    if found["stop"] == "unbounded":
        raise ValueError(f"{WHAT}: the MIP is unbounded, so no plan is within a gap of an optimum")
    if not found["solutions"]:
        if found["stop"] == "limit":
            raise ValueError(f"{WHAT}: the search for the optimum hit max_nodes={max_nodes}; raise max_nodes")
        raise ValueError(f"{WHAT}: the model has no integer plan; use Conflict() to explain why")
    return found["solutions"][0]


def shape(instance, shown, rows, targets, found: dict, xstar: dict, t: float, points: bool) -> dict:
    """The report of variability(): value at x*, min / max (None undecided, +-inf unbounded), argmin / argmax plans with
    points, and exact / bound for an end whose search hit max_nodes."""
    ids = [(v.id, v.index) for v in instance.variables]
    P = instance.precision

    def point(node: Optional[Node]) -> dict:
        at = xstar if node is None else plan_values(node.rhs, node.vrow)
        return {vid: at.get(lab, 0.0) for vid, lab in ids}

    entry: dict = {}
    exact = True
    for k, (lab, s, _) in enumerate(targets):
        side = "max" if s > 0 else "min"
        e = entry.setdefault(lab, {"value": xstar.get(lab, 0.0)})
        state = found["state"][k]
        if state == "unbounded":
            e[side], e["arg" + side] = s * math.inf, None
        elif state == "cycled":
            e[side], e["arg" + side] = None, None
            exact = False
        else:
            e[side] = found["best"][k]
            e["arg" + side] = point(found["witness"][k]) if points else None
        if state == "limit":
            e["exact"] = exact = False
            e.setdefault("bound", {})[side] = found["bound"][k]

    def shaped(lab):
        e = entry[lab]
        d = {"value": e["value"], "min": e["min"], "max": e["max"]}
        if points:
            d["argmin"], d["argmax"] = e["argmin"], e["argmax"]
        if "bound" in e:
            d["exact"], d["bound"] = False, e["bound"]
        return d

    def spread(lab):
        e = entry[lab]
        return math.inf if e["min"] is None or e["max"] is None else e["max"] - e["min"]

    return {"optimum": None, "allowance": t,
            "variables": {v.id: shaped(v.index) for v in shown},
            "constraints": [{"name": cname(c), "type": "max" if c.isUpperBound else "min", "slack": shaped(c.index)}
                            for c in rows],
            "unique": all(spread(v.index) <= P for v in shown), "exact": exact}


def Variability(solver, model: Any, gap=0.0, absolute_gap=0.0, variables=None, constraints=None, points=False,
                max_nodes=10000, width=None, precision: Optional[float] = None, validate: bool = False) -> dict:
    """See the module docstring.  `solver` supplies the engine settings of the tableau (Solver._instance)."""
    if validate:
        model = validation.validate(model)
    if not model:
        raise ValueError("Solver requires a model to operate on")
    _refuse(model)
    opt = model.get("optimize")
    if isinstance(opt, dict):
        key = object_keys(opt)[0]
        model = dict(model, optimize=key, opType="max" if opt[key] == "max" else "min")
    gap, absolute_gap = _gap("gap", gap, WHAT), _gap("absolute_gap", absolute_gap, WHAT)
    max_nodes = pool._count("max_nodes", max_nodes, 1, WHAT)
    width = None if width is None else pool._count("width", width, 1, WHAT)

    instance = solver._instance(model, precision)  # loadJson only: no presolve
    shown, rows = _select(instance, variables, constraints, WHAT)
    it = instance.initial_tableau()
    H, W = it.matrix.shape
    ints = {int(x) for x in it.integerIndices}
    col_of = {int(it.varIndexByCol[c]): c for c in range(1, W)}
    bins = model.get("binaries") or {}
    binaries = {v.index for v in instance.variables if _truthy(bins.get(v.id))}
    search = pool.Search([int(x) for x in it.integerIndices], col_of, binaries)
    targets = targets_of(shown, rows, ints)
    tab, bound = instance.tableau, None
    pivots = 0

    def evaluate_regions(specs):
        nonlocal pivots
        res = tab.pool_batch(specs)
        res["height"] = H
        pivots += int(res["pivots"].sum())
        return [pool._adopt(pool.Region(list(f), list(c)), res, i) for i, (f, c) in enumerate(specs)]

    def evaluate_nodes(specs):
        nonlocal pivots
        res = bound.target_batch([([(1, targets[k][0], float(-targets[k][1]))], c) for k, c in specs],
                                 check_cycles=True)
        pivots += int(res["pivots"].sum())
        return [node_of(res, i, H + 1, c) for i, (_, c) in enumerate(specs)]

    try:
        tab.setModel(instance)
        tab.save()
        launches0 = tab.context.launches
        # rule 1: the optimum and an optimal plan
        found = pool.run(evaluate_regions, search, 1, 0.0, 0.0, max_nodes, pool.DEFAULT_WIDTH if width is None
                         else width)
        best = optimum(found, max_nodes)
        t = allowance(gap, absolute_gap, float(best.rhs[0]))
        xstar = plan_values(best.rhs, best.vrow)
        # rule 2: the bound tableau of the root LP optimum, its allowance widened by what x* loses against it
        tab.restore()
        tab.simplex()
        if tab.lastStatus.cycled:
            raise ValueError(f"{WHAT}: the simplex of the LP relaxation cycled, so there is no optimal tableau to bound")
        lp_raw = float(tab.final_state()[1][0])
        bound = tab.bound(t + max(0.0, float(best.rhs[0]) - lp_raw))
        bound.save()
        wave = iis.wave_width(tab.context, H + 1 + min(len(ints), 8), W)
        out = run(evaluate_nodes, targets, [xstar.get(lab, 0.0) for lab, _, _ in targets], instance.precision,
                  max_nodes, width, wave)
        launches = tab.context.launches - launches0
    finally:
        if bound is not None:
            bound.close()
        tab.close()
    report = shape(instance, shown, rows, targets, out, xstar, t, points)
    sigma = 1.0 if instance.isMinimization else -1.0
    report["optimum"] = sigma * best.evaluation + 0.0
    report.update(searches=len(targets), nodes=found["nodes"] + out["nodes"], lps=found["lps"] + out["lps"],
                  rounds=found["rounds"] + out["rounds"], launches=launches, pivots=pivots)
    return report


def node_of(res: dict, i: int, height: int, cuts) -> Node:
    """Node i of a jslp_target_batch result; column 0 and the labels (height + len(cuts) entries) when integral."""
    node = Node(list(cuts), res["status"][i], res["evaluation"][i], res["is_integral"][i], res["branch_var"][i],
                res["branch_value"][i])
    if node.integral:
        h = height + len(cuts)
        node.rhs, node.vrow = res["rhs"][i, :h].copy(), res["vrow"][i, :h].copy()
    return node

"""Solution pool of a MIP: the k best distinct assignments of its integer and binary variables, best first.  It answers
"which other plans are as good, or nearly as good, as the optimum?", the question variability() answers for LPs.
`Pool(model, k)` takes a JSON model; no earlier solve is needed.  The reference has no counterpart (its keep_solutions
keeps the trail of improving incumbents, which is neither the k best plans nor complete at any gap); DESIGN.md section
2m is the contract.

A solution is an assignment z of the integer variables whose continuous LP (integers fixed at z) is feasible; its value
f(z) is that LP's optimum.  The search is best-first over a partition of the integer assignments into regions: the
model's initial tableau plus fixings (column, value) and bound cuts (type, varIndex, value), the reference's branching
cuts.  Every child region is evaluated when it is created, so a popped region's value bounds everything still open and
an integral region can be emitted when it is popped.  A fractional region splits on its most fractional variable as
branch-and-cut does; an integral region at z is emitted and replaced by the partition of "the region minus z".  Each
round takes the first `width` open regions in pop order and evaluates all their children in one jslp_pool_batch call;
the pops are then committed in true heap order, so `width` changes the LPs solved ("lps"), never the pool.  Presolve
is not run: its fixings zero a cost but leave the column free, which would list copies of one plan."""
from __future__ import annotations

import heapq
import math
import numbers
from typing import Any, Optional

from . import validation
from .model import _truthy, object_keys
from .tableau import EPSILON, js_round
from .variability import _gap

WHAT = "Pool()"
OPTIMAL, INFEASIBLE, UNBOUNDED, CYCLED = 0, 1, 2, 3
DEFAULT_WIDTH = 16


def _count(name: str, x, lo: int, what: str = WHAT) -> int:
    if isinstance(x, bool) or not isinstance(x, numbers.Integral):
        raise ValueError(f"{what}: {name}= takes an integer, not {type(x).__name__}")
    if x < lo:
        raise ValueError(f"{what}: {name}= must be >= {lo}, not {x!r}")
    return int(x)


def _refuse(model: dict) -> None:
    if not (any(_truthy(v) for v in (model.get("ints") or {}).values()) or
            any(_truthy(v) for v in (model.get("binaries") or {}).values())):
        raise ValueError(f"{WHAT} needs integer or binary variables: for a continuous LP use variability()")
    for spec in (model.get("constraints") or {}).values():
        if isinstance(spec, dict) and (spec.get("weight") is not None or spec.get("priority") is not None):
            raise ValueError(f"{WHAT} does not support soft constraints (weight / priority)")
    opt = model.get("optimize")
    if isinstance(opt, dict) and len(object_keys(opt)) > 1:
        raise ValueError(f"{WHAT} takes one objective: `optimize` has {len(object_keys(opt))}")
    if any(_truthy(v) for v in (model.get("unrestricted") or {}).values()):
        raise ValueError(f"{WHAT} does not support unrestricted variables: the exclusion cuts rely on x >= 0")


def replace_cut(cuts: list, cut: tuple) -> list:
    """cuts with `cut` appended, dropping the cuts of the same type on the same variable (branch-and-cut.ts:166-179:
    a `min` cut replaces the variable's `min` cuts and keeps its `max` cuts, and the other way round)."""
    return [c for c in cuts if c[1] != cut[1] or c[0] != cut[0]] + [cut]


class Region:
    """One open region: its fixings and cuts, and its LP's verdict once evaluated."""
    __slots__ = ("fixings", "cuts", "status", "evaluation", "integral", "branch_var", "branch_value", "rhs", "vrow",
                 "children")

    def __init__(self, fixings: list, cuts: list):
        self.fixings, self.cuts = fixings, cuts
        self.children: Optional[list] = None


class Search:
    """The region rules of DESIGN.md section 2m over one model: integer labels in integerIndices order, the column of
    each label, and the binaries (a binary at 1 gets no `min` exclusion cut)."""

    def __init__(self, ints, col_of: dict, binaries: set):
        self.ints, self.col_of, self.binaries = list(ints), col_of, binaries
        self.label_of = {c: lab for lab, c in col_of.items()}

    def fixed_labels(self, region: Region) -> dict:
        return {self.label_of[col]: int(v) for col, v in region.fixings}

    def z_of(self, region: Region) -> dict:
        z = {lab: 0 for lab in self.ints}
        for r in range(1, len(region.vrow)):
            lab = int(region.vrow[r])
            if lab in z:
                z[lab] = int(math.floor(float(region.rhs[r]) + 0.5))
        z.update(self.fixed_labels(region))
        return z

    def children(self, region: Region) -> list:
        """(fixings, cuts) of the regions that replace `region` when it is popped, in push order."""
        if not region.integral:  # branch-and-cut.ts:155-190: cutsHigh, then cutsLow
            v, x = region.branch_var, region.branch_value
            return [(region.fixings, replace_cut(region.cuts, (0, v, float(math.ceil(x))))),
                    (region.fixings, replace_cut(region.cuts, (1, v, float(math.floor(x)))))]
        z, fixed = self.z_of(region), self.fixed_labels(region)
        fixings, cuts, out = list(region.fixings), list(region.cuts), []
        for lab in self.ints:
            if lab in fixed:
                continue
            if z[lab] != 0:
                out.append((fixings, replace_cut(cuts, (1, lab, float(z[lab] - 1)))))
            if not (lab in self.binaries and z[lab] == 1):
                out.append((fixings, replace_cut(cuts, (0, lab, float(z[lab] + 1)))))
            fixings = fixings + [(self.col_of[lab], float(z[lab]))]
            cuts = [c for c in cuts if c[1] != lab]
        return out


def _adopt(region: Region, res: dict, i: int) -> Region:
    region.status = int(res["status"][i])
    region.evaluation = float(res["evaluation"][i])
    region.integral = bool(res["is_integral"][i])
    region.branch_var, region.branch_value = int(res["branch_var"][i]), float(res["branch_value"][i])
    if region.integral:  # the first height + len(cuts) entries are the region's
        h = int(res["height"]) + len(region.cuts)
        region.rhs, region.vrow = res["rhs"][i, :h].copy(), res["vrow"][i, :h].copy()
    return region


def run(evaluate, search: Search, k: int, allowance: float, gap: float, max_nodes: int, width: int) -> dict:
    """The speculative best-first search.  evaluate(list of (fixings, cuts)) -> list of evaluated Regions.  Returns
    {"solutions": [Region...], "stop", "nodes", "lps", "rounds", "allowance"}; "rounds" counts evaluate() calls."""
    heap, seq = [], 0
    sols: list = []
    out = {"stop": None, "nodes": 1, "lps": 1, "rounds": 1}

    def push(r: Region) -> None:
        nonlocal seq
        heapq.heappush(heap, (r.evaluation, -seq, r))  # jslp_frontier.h: lowest first, most recently pushed on ties
        seq += 1

    root = evaluate([([], [])])[0]
    t = None
    if root.status == UNBOUNDED:
        out["stop"] = "unbounded"
    elif root.status == OPTIMAL:
        push(root)
    while out["stop"] is None:
        # commit in true heap order until a popped region has no evaluated children
        while True:
            if not heap:
                out["stop"] = "exhausted"
                break
            top = heap[0][2]
            if sols and top.evaluation > sols[0].evaluation + t:
                out["stop"] = "gap"
                break
            if out["nodes"] >= max_nodes:
                out["stop"] = "limit"
                break
            if top.children is None:
                break
            heapq.heappop(heap)
            if top.integral:
                sols.append(top)
                if len(sols) == 1:
                    t = max(allowance, gap * abs(top.evaluation))
                if len(sols) == k:
                    out["stop"] = "k"
                    break
            out["nodes"] += len(top.children)
            if any(c.status == UNBOUNDED for c in top.children):
                out["stop"] = "unbounded"
                break
            for c in top.children:
                if c.status == OPTIMAL:
                    push(c)
            top.children = []  # committed: its children live in the heap now
        if out["stop"] is not None:
            break
        # speculate: every child of the first `width` open regions in pop order, in one call
        todo = [e[2] for e in heapq.nsmallest(width, heap) if e[2].children is None]
        specs, owner = [], []
        for r in todo:
            ch = search.children(r)
            specs += ch
            owner.append(len(ch))
        done = evaluate(specs) if specs else []
        out["lps"] += len(specs)
        out["rounds"] += 1
        pos = 0
        for r, n in zip(todo, owner):
            r.children = done[pos:pos + n]
            pos += n
    out["solutions"] = sols
    out["allowance"] = t
    return out


def Pool(solver, model: Any, k=10, gap=0.0, absolute_gap=0.0, precision: Optional[float] = None,
         validate: bool = False, max_nodes=100000, width=None) -> dict:
    """See the module docstring.  `solver` supplies the engine settings of the tableau (Solver._instance)."""
    if validate:
        model = validation.validate(model)
    if not model:
        raise ValueError("Solver requires a model to operate on")
    if not isinstance(model, dict):
        raise ValueError(f"{WHAT} takes a JSON model")
    if model.get("external"):
        raise ValueError(f"{WHAT} does not support external solvers")
    _refuse(model)
    opt = model.get("optimize")
    if isinstance(opt, dict):
        key = object_keys(opt)[0]
        model = dict(model, optimize=key, opType="max" if opt[key] == "max" else "min")
    k = _count("k", k, 1)
    max_nodes = _count("max_nodes", max_nodes, 1)
    width = DEFAULT_WIDTH if width is None else _count("width", width, 1)
    gap, absolute_gap = _gap("gap", gap, WHAT), _gap("absolute_gap", absolute_gap, WHAT)

    instance = solver._instance(model, precision)  # loadJson only: no presolve
    it = instance.initial_tableau()
    col_of = {int(it.varIndexByCol[c]): c for c in range(1, it.matrix.shape[1])}
    bins = model.get("binaries") or {}
    binaries = {v.index for v in instance.variables if _truthy(bins.get(v.id))}
    search = Search([int(x) for x in it.integerIndices], col_of, binaries)
    tab = instance.tableau
    height = it.matrix.shape[0]

    pivots = 0

    def evaluate(specs):
        nonlocal pivots
        res = tab.pool_batch(specs)
        res["height"] = height
        pivots += int(res["pivots"].sum())
        return [_adopt(Region(list(f), list(c)), res, i) for i, (f, c) in enumerate(specs)]

    try:
        tab.setModel(instance)
        tab.save()
        launches0 = tab.context.launches
        found = run(evaluate, search, k, absolute_gap, gap, max_nodes, width)
        launches = tab.context.launches - launches0
    finally:
        tab.close()
    sigma = 1.0 if instance.isMinimization else -1.0
    rounding = js_round(1 / instance.precision)
    ints = set(search.ints)
    solutions = []
    for rank, r in enumerate(found["solutions"], start=1):
        z = search.z_of(r)
        row_of = {int(r.vrow[i]): i for i in range(1, len(r.vrow))}
        values = {}
        for v in instance.variables:
            if v.index in ints:
                values[v.id] = float(z[v.index])
            elif v.index in row_of:
                values[v.id] = js_round((EPSILON + float(r.rhs[row_of[v.index]])) * rounding) / rounding
            else:
                values[v.id] = 0.0
        solutions.append({"result": sigma * r.evaluation + 0.0, "values": values, "rank": rank})
    return {"solutions": solutions, "optimum": solutions[0]["result"] if solutions else None,
            "allowance": found["allowance"], "stop": found["stop"], "nodes": found["nodes"], "lps": found["lps"],
            "rounds": found["rounds"], "launches": launches, "pivots": pivots}

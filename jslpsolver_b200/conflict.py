"""Conflict of an infeasible MIP: a set of constraint rows and integrality restrictions that has no integer plan as a
whole, and has one once any single member is dropped.  It answers "why does my model have no integer plan?" when the
LP relaxation has one (a schedule whose shift sizes cannot add up, a Sudoku with contradictory givens), which an LP IIS
cannot: in 2x + 2y = 3 the rows conflict only through integrality.  The reference has no counterpart; DESIGN.md
section 2n is the contract.

Every membership test is test(S, J): is there a plan of the rows S that is integral on the labels J?  It is a
depth-first branch and bound over phase-1 node LPs (a node is a list of the reference's branching cuts).  The rows are
filtered first, with integrality on every label, then the labels with the rows fixed, both by iis.deletion_filter; a
filter round's tests run as concurrent searches, and each step evaluates the top `depth` unevaluated entries of every
live search's stack in one jslp_conflict_batch call.  Each search commits its results in stack order, so `width` and
`depth` change the LPs solved ("lps"), never the answer.  Presolve is not run: the answer describes the model as
written.  Variable non-negativity is implicit, as in iis()."""
from __future__ import annotations

import math
import numbers
from typing import Any, Optional

import numpy as np

from . import iis, validation
from .model import _truthy, object_keys
from .pool import replace_cut

WHAT = "Conflict()"
FEASIBLE, INFEASIBLE, UNDECIDED = iis.FEASIBLE, iis.INFEASIBLE, iis.UNDECIDED
NODE_FEASIBLE, NODE_INFEASIBLE, NODE_CYCLED = 0, 1, 2  # jslp_conflict_batch's status


def _count(name: str, x, lo: int) -> int:
    if isinstance(x, bool) or not isinstance(x, numbers.Integral):
        raise ValueError(f"{WHAT}: {name}= takes an integer, not {type(x).__name__}")
    if x < lo:
        raise ValueError(f"{WHAT}: {name}= must be >= {lo}, not {x!r}")
    return int(x)


def refuse(model: Any) -> None:
    """The models Conflict() does not explain, as ValueError."""
    if not isinstance(model, dict):
        raise ValueError(f"{WHAT} takes a JSON model")
    if model.get("external"):
        raise ValueError(f"{WHAT} does not support external solvers")
    opt = model.get("optimize")
    if isinstance(opt, dict) and len(object_keys(opt)) > 1:
        raise ValueError(f"{WHAT} takes one objective: `optimize` has {len(object_keys(opt))}")
    for spec in (model.get("constraints") or {}).values():
        if isinstance(spec, dict) and (spec.get("weight") is not None or spec.get("priority") is not None):
            raise ValueError(f"{WHAT} does not support soft constraints (weight / priority)")
    if not (any(_truthy(v) for v in (model.get("ints") or {}).values()) or
            any(_truthy(v) for v in (model.get("binaries") or {}).values())):
        raise ValueError(f"{WHAT} needs integer or binary variables: for a continuous LP use "
                         "Solve(model, full=True).iis()")


class Node:
    """One evaluated node LP: status (NODE_*), is_integral on the test's labels, branching variable and value, phase-1
    pivots, and column 0 with the row labels (None when the node cycled)."""
    __slots__ = ("status", "integral", "branch_var", "branch_value", "pivots", "rhs", "vrow")

    def __init__(self, status, integral, branch_var, branch_value, pivots, rhs=None, vrow=None):
        self.status, self.integral = int(status), bool(integral)
        self.branch_var, self.branch_value, self.pivots = int(branch_var), float(branch_value), int(pivots)
        self.rhs, self.vrow = rhs, vrow


def children(cuts: list, node: Node) -> list:
    """The cut lists of a fractional node's children in push order: the `min ceil(x)` child, then the `max floor(x)`
    child, each replacing the same-type cut on the branching variable (branch-and-cut.ts:155-190)."""
    v, x = node.branch_var, node.branch_value
    return [replace_cut(cuts, (0, v, float(math.ceil(x)))), replace_cut(cuts, (1, v, float(math.floor(x))))]


class _Search:
    __slots__ = ("rows", "ints", "stack", "nodes", "cycled", "verdict", "witness")

    def __init__(self, rows, ints):
        self.rows, self.ints = list(rows), list(ints)
        self.stack = [[[], None]]  # [cuts, Node once evaluated]; the top is the last entry
        self.nodes, self.cycled = 0, False
        self.verdict, self.witness = None, None

    def commit(self, max_nodes: int) -> None:
        """Pops the evaluated entries at the top of the stack in order, as the sequential search would."""
        while self.verdict is None and self.stack and self.stack[-1][1] is not None:
            cuts, node = self.stack.pop()
            self.nodes += 1
            if node.status == NODE_CYCLED:
                self.cycled = True
            elif node.status == NODE_FEASIBLE:
                if node.integral:
                    self.verdict, self.witness = FEASIBLE, node
                    return
                self.stack += [[c, None] for c in children(cuts, node)]
            if not self.stack:
                self.verdict = UNDECIDED if self.cycled else INFEASIBLE
            elif self.nodes >= max_nodes:
                self.verdict = UNDECIDED


def run(evaluate, tests, max_nodes: int, depth: Optional[int] = None, wave: int = 1):
    """The concurrent searches of tests = [(rows, labels), ...].  evaluate([(rows, labels, cuts), ...]) -> [Node, ...].
    Each step takes the top `depth` unevaluated entries of every live search's stack (depth None: wave // live
    searches, at least 1) into one evaluate() call, then commits every search in stack order.  Returns ([(verdict,
    witness Node or None), ...], {"nodes": committed nodes, "lps": evaluated nodes, "calls": evaluate() calls})."""
    searches = [_Search(r, j) for r, j in tests]
    count = {"nodes": 0, "lps": 0, "calls": 0}
    live = list(searches)
    while live:
        d = depth if depth is not None else max(1, wave // len(live))
        specs, slots = [], []
        for s in live:
            picked = 0
            for e in reversed(s.stack):
                if picked == d:
                    break
                if e[1] is None:
                    specs.append((s.rows, s.ints, e[0]))
                    slots.append(e)
                    picked += 1
        for e, node in zip(slots, evaluate(specs)):
            e[1] = node
        count["lps"] += len(specs)
        count["calls"] += 1
        for s in live:
            s.commit(max_nodes)
        live = [s for s in live if s.verdict is None]
    count["nodes"] = sum(s.nodes for s in searches)
    return [(s.verdict, s.witness) for s in searches], count


class Tests:
    """test(S, J) over one evaluate(), with every verdict and witness kept by (S, J) and the counters summed."""

    def __init__(self, evaluate, max_nodes: int, depth: Optional[int], wave: int):
        self.evaluate, self.max_nodes, self.depth, self.wave = evaluate, max_nodes, depth, wave
        self.done: dict = {}
        self.count = {"tests": 0, "nodes": 0, "lps": 0, "calls": 0}

    def __call__(self, tests) -> list:
        keys = [(tuple(r), tuple(j)) for r, j in tests]
        todo = list(dict.fromkeys(k for k in keys if k not in self.done))
        if todo:
            out, c = run(self.evaluate, todo, self.max_nodes, self.depth, self.wave)
            self.done.update(zip(todo, out))
            self.count["tests"] += len(todo)
            for k in ("nodes", "lps", "calls"):
                self.count[k] += c[k]
        return [self.done[k] for k in keys]


def committed_set(order: list, kept: list, member) -> list:
    """The set the sequential deletion filter over `order` tested to decide `member`, which it kept: the kept items
    before it and every item after it."""
    at, keep = order.index(member), set(kept)
    return [x for i, x in enumerate(order) if (x in keep and i < at) or i > at]


def search(test: Tests, rows: list, ints: list, relaxation: int, support, width: int, prepass: bool = True) -> dict:
    """The start and both filters of DESIGN.md section 2n.  relaxation = the LP verdict of every row; support = the
    rows of its phase-1 certificate when it is INFEASIBLE.  Returns {"rows", "ints", "irreducible", "row_witness",
    "int_witness"} with the witnesses by member (None for a member kept on an undecided test)."""
    verdict = test([(rows, ints)])[0][0]
    if verdict == FEASIBLE:
        raise ValueError(f"{WHAT}: the model has an integer plan, so there is no conflict to explain")
    if verdict == UNDECIDED:
        raise ValueError(f"{WHAT}: the search over the whole model is undecided within max_nodes "
                         "(or a node LP cycled); raise max_nodes")
    S0 = rows
    if relaxation == INFEASIBLE and support != rows and test([(support, ints)])[0][0] == INFEASIBLE:
        S0 = list(support)
    B, irr_rows = iis.deletion_filter(lambda sets: [v for v, _ in test([(s, ints) for s in sets])], S0, width, prepass)
    J, irr_ints = [], True
    if test([(B, [])])[0][0] != INFEASIBLE:
        J, irr_ints = iis.deletion_filter(lambda sets: [v for v, _ in test([(B, s) for s in sets])], ints, width,
                                          prepass)
    row_witness = {r: test([([x for x in committed_set(S0, B, r)], ints)])[0][1] for r in B}
    int_witness = {j: test([(B, committed_set(ints, J, j))])[0][1] for j in J}
    return {"rows": B, "ints": J, "irreducible": irr_rows and irr_ints, "row_witness": row_witness,
            "int_witness": int_witness}


def plan(node: Optional[Node], ids: dict) -> Optional[dict]:
    """{"values": {id: value}} of a witness node: column 0 of the row each structural variable is basic in, 0 for
    the non-basic ones."""
    if node is None:
        return None
    at = {int(node.vrow[r]): float(node.rhs[r]) for r in range(1, len(node.vrow))}
    return {"values": {vid: at.get(lab, 0.0) for lab, vid in ids.items()}}


def Conflict(solver, model: Any, max_nodes=10000, width=None, depth=None, precision: Optional[float] = None,
             validate: bool = False) -> dict:
    """See the module docstring.  `solver` supplies the engine settings of the tableau (Solver._instance)."""
    if validate:
        model = validation.validate(model)
    if not model:
        raise ValueError("Solver requires a model to operate on")
    refuse(model)
    opt = model.get("optimize")
    if isinstance(opt, dict):
        key = object_keys(opt)[0]
        model = dict(model, optimize=key, opType="max" if opt[key] == "max" else "min")
    max_nodes = _count("max_nodes", max_nodes, 1)
    width = None if width is None else _count("width", width, 1)
    depth = None if depth is None else _count("depth", depth, 1)

    instance = solver._instance(model, precision)  # loadJson only: no presolve
    it = instance.initial_tableau()
    H, W = it.matrix.shape
    rows = list(range(1, H))
    ints = [int(x) for x in it.integerIndices]
    pos_of = {lab: p for p, lab in enumerate(ints)}
    ids = {v.index: v.id for v in instance.variables}
    tab = instance.tableau
    pivots = 0

    def evaluate(specs):
        nonlocal pivots
        keep = np.zeros((len(specs), H), dtype=np.uint8)
        int_keep = np.zeros((len(specs), len(ints)), dtype=np.uint8)
        for i, (S, J, _) in enumerate(specs):
            keep[i, list(S)] = 1
            int_keep[i, [pos_of[j] for j in J]] = 1
        res = tab.conflict_batch(keep, int_keep, [c for _, _, c in specs])
        pivots += int(res["pivots"].sum())
        out = []
        for i, (S, _, c) in enumerate(specs):
            h = 1 + len(S) + len(c)
            cycled = res["status"][i] == NODE_CYCLED
            out.append(Node(res["status"][i], res["is_integral"][i], res["branch_var"][i], res["branch_value"][i],
                            res["pivots"][i], None if cycled else res["rhs"][i, :h].copy(),
                            None if cycled else res["vrow"][i, :h].copy()))
        return out

    try:
        tab.setModel(instance)
        tab.save()
        launches0 = tab.context.launches
        relaxation = int(tab.feasibility_batch(np.ones((1, H), dtype=np.uint8))[0][0])
        support = None
        if relaxation == INFEASIBLE:
            tab.phase1()
            support = iis.certificate_support(tab.matrix2d(), tab.varIndexByRow, tab.varIndexByCol,
                                              instance.precision, {int(it.varIndexByRow[r]): r for r in rows})
            tab.restore()
        # room for the cut rows of an 8-level dive; taller nodes run on the single-tableau path either way
        wave = iis.wave_width(tab.context, H + min(len(ints), 8), W)
        test = Tests(evaluate, max_nodes, depth, wave)
        found = search(test, rows, ints, relaxation, support, wave if width is None else width)
        launches = tab.context.launches - launches0
    finally:
        tab.close()
    constraints, bounds, names = [], [], []
    for r in found["rows"]:
        con = instance.constraints[r - 1]
        witness = plan(found["row_witness"][r], ids)
        if con.name is None:  # the `x <= 1` row loadJson adds for a binary (model.ts:392-395)
            var = next(iter(con.coef.values())).variable
            bounds.append({"variable": var.id, "type": "max", "rhs": 1, "witness": witness})
            continue
        constraints.append({"name": con.name, "type": "max" if con.isUpperBound else "min", "rhs": con.rhs,
                            "witness": witness})
        if con.name not in names:
            names.append(con.name)
    integers = [{"variable": ids[j], "witness": plan(found["int_witness"][j], ids)} for j in found["ints"]]
    return {"constraints": constraints, "bounds": bounds, "integers": integers, "names": names,
            "relaxation": {INFEASIBLE: "infeasible", FEASIBLE: "feasible"}.get(relaxation, "undecided"),
            "irreducible": found["irreducible"], "tests": test.count["tests"], "nodes": test.count["nodes"],
            "lps": test.count["lps"], "launches": launches, "pivots": pivots}

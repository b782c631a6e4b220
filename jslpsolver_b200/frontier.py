"""The Pareto frontier of a continuous LP with two objectives: every efficient vertex between the optimum of the first
objective and the optimum of the second, each with the interval of weights that selects it.  `Frontier(model)` takes
the JSON model `MultiObjective` takes, with exactly two keys in `optimize`.  The reference has no counterpart (its
Polyopt returns the two ends and a midpoint that need not be efficient); DESIGN.md section 2g is the contract.

For an LP the frontier is a concave piecewise-linear curve whose vertices are the optima of (1 - w) * g1 + w * g2 as
the weight w goes from 0 to 1, where gk is objective k with its sense applied.  The model is solved for the first
objective as Solve() solves it; the device then prices the second objective against that optimal basis and moves w
with one primal simplex pivot per basis change (jslp_frontier), returning every point it passes.  This module loads
and checks the model, builds the second objective's row, and turns the points into vertices."""
from __future__ import annotations

from typing import Any, Optional

from . import validation
from .model import _truthy, object_keys

STOPS = {1: "reached", 3: "unbounded", 4: "limit"}
WHAT = "Frontier()"


def _objectives(model: dict):
    opt = model.get("optimize")
    keys = object_keys(opt) if isinstance(opt, dict) else []
    if len(keys) != 2:
        raise ValueError(f"{WHAT} needs `optimize` with exactly two objectives, e.g. {{\"a\": \"max\", \"b\": \"min\"}}")
    return keys, {k: "max" if opt[k] == "max" else "min" for k in keys}


def _refuse(model: dict, what: str = WHAT) -> None:
    if any(_truthy(v) for v in (model.get("ints") or {}).values()) or \
            any(_truthy(v) for v in (model.get("binaries") or {}).values()):
        raise ValueError(f"{what} is defined for continuous LPs only: the model has integer or binary variables")
    for spec in (model.get("constraints") or {}).values():
        if isinstance(spec, dict) and (spec.get("weight") is not None or spec.get("priority") is not None):
            raise ValueError(f"{what} does not support soft constraints (weight / priority)")


def _coef(jm: dict, vid: str, key: str) -> float:
    c = jm["variables"][vid].get(key)
    return float(c) if _truthy(c) else 0.0


def cost_row(m, jm: dict, key: str, sense: str, n_labels: int) -> list:
    """C2 by label: sigma2 * c2_j at each structural variable's label (the sign initial_tableau gives row 0), 0 for
    slacks and for variables that presolve fixed."""
    sigma = 1.0 if sense == "max" else -1.0
    fixed = m.presolveResult.fixedVariables if m.presolveResult is not None else {}
    c2 = [0.0] * n_labels
    for v in m.variables:
        if v not in fixed:
            c2[v.index] = sigma * _coef(jm, v.id, key)
    return c2


def vertices(points, starts, end, stop, precision):
    """The vertex rule of section 2g.  points[k] = the structural values of the k-th distinct point in path order and
    starts[k] the weight where it starts; the last one stands until `end`.  Neighbouring equal points merge.  A point
    whose interval is no longer than the precision drops out (the first objective's other optima passed at weight 0,
    collinear points inside an edge, and pivots that rounding lets through next to a breakpoint); its weights go to
    the next vertex kept, or to the last one at the end.  The final point of an unbounded path stays."""
    segs = []
    for k, pt in enumerate(points):
        to = starts[k + 1] if k + 1 < len(points) else end
        if segs and segs[-1][0] == pt:
            segs[-1][2] = to
        else:
            segs.append([pt, starts[k], to])
    out, pending = [], None
    for k, (pt, lo, hi) in enumerate(segs):
        if hi - lo > precision or (stop == "unbounded" and k == len(segs) - 1):
            lo = lo if pending is None else pending
            pending = None
            if out and out[-1][0] == pt:
                out[-1][2] = hi
            else:
                out.append([pt, lo, hi])
        elif pending is None:
            pending = lo
    if pending is not None:
        if out:
            out[-1][2] = segs[-1][2]
        else:
            out.append([segs[-1][0], pending, segs[-1][2]])
    return [tuple(s) for s in out]


def objective_sums(m, jm: dict, keys, pt) -> dict:
    """{key: the sum of c_key,j * x_j in variable order} at the point pt (structural values in m.variables order)."""
    objs = {}
    for key in keys:
        acc = 0.0
        for v, x in zip(m.variables, pt):
            acc += _coef(jm, v.id, key) * x
        objs[key] = acc
    return objs


def result(m, jm: dict, keys, senses, out) -> dict:
    """The Frontier() result from a frontier_path() output on the tableau of model `m` (loaded from `jm`)."""
    fixed = m.presolveResult.fixedVariables if m.presolveResult is not None else {}
    theta = [float(x) for x in out["theta"]]
    stop = STOPS[int(out["stop"])]
    end = theta[-1] if theta else 0.0
    points, starts = [], []
    for rhs, vrow, at in zip(out["pt_rhs"], out["pt_vrow"], out["pt_break"]):
        row_of = {int(vrow[r]): r for r in range(1, len(vrow))}
        points.append(tuple(fixed[v] if v in fixed else (float(rhs[row_of[v.index]]) if v.index in row_of else 0.0)
                            for v in m.variables))
        starts.append(0.0 if int(at) == 0 else theta[int(at) - 1])
    out_v = []
    for pt, lo, hi in vertices(points, starts, end, stop, m.precision):
        values = {v.id: x for v, x in zip(m.variables, pt)}
        out_v.append({"weight": {"from": lo, "to": hi}, "objectives": objective_sums(m, jm, keys, pt),
                      "values": values})
    pivots = sum(1 for r in out["rc_lbl"] if int(r[0]) >= 0 and int(r[1]) >= 0)
    return {"feasible": True, "objectives": dict(senses), "vertices": out_v, "stop": stop, "end": end,
            "pivots": pivots}


def Frontier(solver, model: Any, precision: Optional[float] = None, validate: bool = False) -> dict:
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
    _refuse(model)
    first, second = keys
    working = dict(model, optimize=first, opType=senses[first])
    instance = solver._instance(working, precision)
    solution = instance.solve()
    if not solution.feasible:
        return {"feasible": False, "objectives": dict(senses), "vertices": [], "stop": None, "end": None, "pivots": 0}
    if not solution.bounded:
        raise ValueError(f"{WHAT}: the first objective {first!r} is unbounded; list the objectives the other way round "
                         f"(optimize = {{{second!r}: {senses[second]!r}, {first!r}: {senses[first]!r}}}): the path from "
                         "the bounded end then stops with stop = 'unbounded'")
    t = instance.tableau
    c2 = cost_row(instance, working, second, senses[second], t.nVars)
    out = t.frontier_path(c2, 4 * (t.height + t.width))
    return result(instance, working, keys, senses, out)

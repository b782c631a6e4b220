"""The Pareto frontier of a MIP with two objectives: every nondominated image (f1, f2) over the integer plans, in
frontier order from the first objective's lexicographic optimum to the second's.  It answers "what does each unit of
the second objective cost in the first?" for models with `ints` / `binaries`, the question Frontier() answers for
continuous LPs.  `FrontierMIP(model)` takes the JSON model Frontier() takes, with `ints` or `binaries`.  The reference
has no counterpart; DESIGN.md section 2s is the contract.

A MIP frontier is not convex, so no weighted sum of the objectives reaches its unsupported points.  This is the
balanced box method (Boland, Charkhgard and Savelsbergh, 2015).  With gk = sigma_k * f_k (both minimised), the ends are
a = lexmin(g1, g2) and b = lexmin(g2, g1), each a LexicographicMIP() chain at gap 0 (lexicographic_mip.chain).  Every
box between two known points a (top left) and b (bottom right) then takes four exact searches at most: c =
lexmin(g1, g2) under g1 <= b1 - step, g2 <= (a2 + b2) / 2, and d = lexmin(g2, g1) under g1 <= c1 - step,
g2 <= a2 - step; c and d are new frontier points, and the boxes (a, d) and (c, b) are left.  Every search is a node
LP of one box tableau, the model's initial tableau with the two rows g1 <= u1 and g2 <= u2, uploaded once: the bounds
are right-hand-side edits of the two rows, a g2 search adds the cost edits that turn row 0 from g1 into g2, and the
branching cuts follow (jslp_box_batch).  Each stage advances every live box by one search, all of them concurrent
targets of mip_variability.run in shared launches.  The model is loaded as LexicographicMIP() loads it (no presolve,
no tolerance / timeout), so the answer describes the model as written, up to the node and point limits."""
from __future__ import annotations

import math
import numbers
from typing import Any, Optional

from . import iis, pool, validation
from .frontier import _coef, objective_sums
from .lexicographic_mip import OWN, chain
from .mip_variability import node_of, plan_values, refuse_non_mip, refuse_unrestricted, run
from .model import _truthy, object_keys

WHAT = "FrontierMIP()"


def objectives(model: Any) -> tuple:
    """The refusals of section 2s in order, then (keys, senses)."""
    if not isinstance(model, dict):
        raise ValueError(f"{WHAT} takes a JSON model")
    if model.get("external"):
        raise ValueError(f"{WHAT} does not support external solvers")
    opt = model.get("optimize")
    keys = object_keys(opt) if isinstance(opt, dict) else []
    if len(keys) != 2:
        raise ValueError(f"{WHAT} needs `optimize` with exactly two objectives, e.g. {{\"a\": \"max\", \"b\": \"min\"}}")
    refuse_non_mip(model, WHAT, "Frontier()")
    refuse_unrestricted(model, WHAT)
    integer = {vid for vid in model["variables"]
               if _truthy((model.get("ints") or {}).get(vid)) or _truthy((model.get("binaries") or {}).get(vid))}
    for key in keys:
        for vid in object_keys(model["variables"]):
            if vid not in integer and _coef(model, vid, key) != 0.0:
                raise ValueError(f"{WHAT}: objective {key!r} has a nonzero coefficient on the continuous variable "
                                 f"{vid!r}; with continuous variables in an objective the frontier has segments "
                                 "between its points, which this search does not trace")
    return keys, {k: "max" if opt[k] == "max" else "min" for k in keys}


def step_of(model: dict, keys, step) -> tuple:
    """(step, proven): step=None is 1 when every objective coefficient is an integer, and must be given otherwise.
    `proven` is True when every coefficient is an integer multiple of step, so that two distinct values of an objective
    over integer plans differ by at least step and no nondominated point can be missed."""
    coefs = [_coef(model, vid, key) for key in keys for vid in object_keys(model["variables"])]
    if step is None:
        if not all(float(c).is_integer() for c in coefs):
            raise ValueError(f"{WHAT}: an objective has non-integer coefficients, so step= must be given: the least "
                             "difference in each objective between two distinct frontier points")
        step = 1.0
    elif isinstance(step, bool) or not isinstance(step, numbers.Real) or not math.isfinite(step) or step <= 0:
        raise ValueError(f"{WHAT}: step= must be a finite number > 0, not {step!r}")
    step = float(step)
    return step, all(float(c / step).is_integer() for c in coefs)


def fresh_names(model: dict, n: int) -> list:
    """n attribute names used by no constraint, no variable attribute and no objective of the model."""
    used = set(model.get("constraints") or {}) | set(model.get("optimize") or {})
    for attrs in model["variables"].values():
        used |= set(attrs)
    out, k = [], 0
    while len(out) < n:
        name = f"frontier.{k}"
        k += 1
        if name not in used:
            out.append(name)
    return out


def loads(model: dict, keys, senses: dict) -> dict:
    """The JSON models of section 2s rule 1: "first" and "second" (the objectives under fresh names o1 / o2, chains
    lexmin(g1, g2) and lexmin(g2, g1)), and "box" ("first" with the rows r1: g1 <= 0 and r2: g2 <= 0).  Each variable
    loses its keys[0] attribute, so a constraint named like keys[0] has no terms in any of them, as LexicographicMIP()
    and Frontier() load the model; "names" = (o1, o2, r1, r2)."""
    o1, o2, r1, r2 = fresh_names(model, 4)
    sigma = {k: 1.0 if senses[k] == "min" else -1.0 for k in keys}
    base, box = {}, {}
    for vid in object_keys(model["variables"]):
        attrs = {a: x for a, x in model["variables"][vid].items() if a != keys[0]}
        c1, c2 = _coef(model, vid, keys[0]), _coef(model, vid, keys[1])
        attrs.update({o: c for o, c in ((o1, c1), (o2, c2)) if c != 0.0})
        base[vid] = attrs
        box[vid] = dict(attrs, **{r: s * c for r, s, c in ((r1, sigma[keys[0]], c1), (r2, sigma[keys[1]], c2))
                                  if c != 0.0})
    first = dict(model, variables=base, optimize=o1, opType=senses[keys[0]])
    second = dict(model, variables=base, optimize=o2, opType=senses[keys[1]])
    rows = dict(model.get("constraints") or {}, **{r1: {"max": 0}, r2: {"max": 0}})
    return {"first": first, "second": second, "box": dict(first, variables=box, constraints=rows),
            "names": (o1, o2, r1, r2)}


def point(instance, model: dict, keys, senses: dict, plan: tuple) -> dict:
    """A frontier point of the plan (structural values in instance.variables order): its values, with every integer
    variable at the integer its value rounds to (the integrality scan accepted it within the precision), and from them
    its objectives and image g = (g1, g2).  Only integer variables enter an objective, so the image is exact for integer
    coefficients and the box bounds built from it cut no plan off by rounding."""
    plan = tuple(float(math.floor(x + 0.5)) if v.isInteger else x for v, x in zip(instance.variables, plan))
    f = objective_sums(instance, model, keys, plan)
    g = tuple((1.0 if senses[k] == "min" else -1.0) * f[k] for k in keys)
    return {"objectives": f, "values": {v.id: x for v, x in zip(instance.variables, plan)}, "g": g}


def box_edits(instance, model: dict, keys, senses: dict, rows) -> tuple:
    """(slack labels of the rows r1 / r2 of the box tableau, the cost edits [(1, label, g2_j - g1_j), ...] of a g2
    search, nonzero differences only, in variable order)."""
    slack = {c.name: c.index for c in instance.constraints if c.name in rows}
    s1, s2 = (1.0 if senses[k] == "min" else -1.0 for k in keys)
    cost = []
    for v in instance.variables:
        d = s2 * _coef(model, v.id, keys[1]) - s1 * _coef(model, v.id, keys[0])
        if d != 0.0:
            cost.append((1, v.index, d))
    return (slack[rows[0]], slack[rows[1]]), cost


def node_spec(slack, cost, u1: float, u2: float, k: int) -> list:
    """The edits of one box search: g1 <= u1 and g2 <= u2 (updateRightHandSide of rows written with max 0), then for
    k = 1 the cost edits of g2."""
    return [(0, slack[0], -u1), (0, slack[1], -u2)] + (cost if k == 1 else [])


class Box:
    """A box between two known frontier points a (top left) and b (bottom right), and how far rule 3 has got in it:
    phase L1 / L2 (the lower stage's two searches), U1 / U2 (the upper stage's)."""
    __slots__ = ("a", "b", "phase", "low", "c", "up")

    def __init__(self, a: dict, b: dict):
        self.a, self.b, self.phase, self.low, self.c, self.up = a, b, "L1", None, None, None

    def spec(self, step: float, P: float) -> tuple:
        """(u1, u2, k) of the next search: g1 <= u1, g2 <= u2, minimising g1 (k = 0) or g2 (k = 1)."""
        m = (self.a["g"][1] + self.b["g"][1]) / 2
        if self.phase == "L1":
            return self.b["g"][0] - step, m, 0
        if self.phase == "L2":
            return self.low["g"][0] + P, m, 1
        if self.phase == "U1":
            return self.c["g"][0] - step, self.a["g"][1] - step, 1
        return self.c["g"][0] - step, self.up["g"][1] + P, 0

    def advance(self, found: Optional[dict]):
        """Takes the point of an exact search (None: no plan).  Returns None while the box is live, else (new points
        in frontier order, new boxes in frontier order)."""
        if self.phase == "L1":
            if found is None:
                self.c, self.phase = self.b, "U1"
            else:
                self.low, self.phase = found, "L2"
            return None
        if found is None and self.phase in ("L2", "U2"):
            raise RuntimeError(f"{WHAT}: the second search of a stage has no integer plan, but the first found one")
        if self.phase == "L2":
            self.c, self.phase = found, "U1"
            return None
        if self.phase == "U1" and found is not None:
            self.up, self.phase = found, "U2"
            return None
        d = self.a if found is None else found
        new = [p for p, known in ((d, self.a), (self.c, self.b)) if p is not known]
        boxes = ([Box(self.a, d)] if d is not self.a else []) + ([Box(self.c, self.b)] if self.c is not self.b else [])
        return new, boxes


def trace(a: dict, b: dict, step: float, P: float, max_points: int, stage) -> dict:
    """Rules 3 and 4: the boxes from (a, b) until none is live.  stage(specs) runs one exact search per spec (u1, u2, k)
    as concurrent targets and returns [(state, point or None)] in spec order.  A box whose search ends "limit" or
    "cycled", or whose points would pass max_points, goes to open whole; once the points reach max_points every live
    box does.  Returns {"points" (a and b included, unordered), "open", "stop", "searches"}."""
    points, opened, live = [a, b], [], [Box(a, b)]
    stop, searches = "reached", 0
    while live:
        if len(points) >= max_points:
            opened += live
            stop = stop if stop == "cycled" else "limit"
            break
        results = stage([box.spec(step, P) for box in live])
        searches += len(live)
        nxt = []
        for box, (state, found) in zip(live, results):
            if state == "unbounded":
                raise RuntimeError(f"{WHAT}: a box search came out unbounded, but both ends of the frontier are bounded")
            if state in ("limit", "cycled"):
                opened.append(box)
                stop = "cycled" if "cycled" in (state, stop) else "limit"
                continue
            done = box.advance(found)
            if done is None:
                nxt.append(box)
            elif len(points) + len(done[0]) > max_points:
                opened.append(box)
                stop = stop if stop == "cycled" else "limit"
            else:
                points += done[0]
                nxt += done[1]
        live = nxt
    return {"points": points, "open": opened, "stop": stop, "searches": searches}


def same_image(p: dict, q: dict, P: float) -> bool:
    return abs(p["g"][0] - q["g"][0]) <= P and abs(p["g"][1] - q["g"][1]) <= P


def result(keys, senses: dict, step: float, proven: bool, ends, traced: Optional[dict], stop, P: float) -> dict:
    """The FrontierMIP() result without its counters: ends = the points of the two chains that were reached."""
    points = traced["points"] if traced is not None else [p for p in ends if p is not None]
    if traced is None and len(points) == 2 and same_image(points[0], points[1], P):
        points = points[:1]
    points = sorted(points, key=lambda p: p["g"][0])
    opened = sorted(traced["open"], key=lambda box: box.a["g"][0]) if traced is not None else []
    return {"feasible": True, "bounded": stop != "unbounded", "stop": stop,
            "exact": stop == "reached" and proven, "objectives": dict(senses), "step": step,
            "points": [{"objectives": p["objectives"], "values": p["values"]} for p in points],
            "open": [{"from": box.a["objectives"], "to": box.b["objectives"]} for box in opened]}


def no_plan(key: str, max_nodes: int) -> str:
    return (f"{WHAT}: the search for the optimum of {key!r} hit max_nodes={max_nodes} before any integer plan; raise "
            "max_nodes")


def ends_stop(ra: dict, rb: Optional[dict]) -> Optional[str]:
    """The stop of the two chains when either did not reach its end: unbounded first, then cycled, then limit."""
    stops = [r["stop"] for r in (ra, rb) if r is not None]
    for s in ("unbounded", "cycled", "limit"):
        if s in stops:
            return s
    return None


def FrontierMIP(solver, model: Any, *, step=None, max_points=1000, max_nodes=10000, width=None,
                precision: Optional[float] = None, validate: bool = False) -> dict:
    """See the module docstring.  `solver` supplies the engine settings of the tableaux (Solver._instance)."""
    if validate:
        model = validation.validate(model)
    if not model:
        raise ValueError("Solver requires a model to operate on")
    keys, senses = objectives(model)
    step, proven = step_of(model, keys, step)
    max_points = pool._count("max_points", max_points, 2, WHAT)
    max_nodes = pool._count("max_nodes", max_nodes, 1, WHAT)
    width = None if width is None else pool._count("width", width, 1, WHAT)
    jm = loads(model, keys, senses)
    o1, o2, r1, r2 = jm["names"]
    osenses = {o1: senses[keys[0]], o2: senses[keys[1]]}
    count = {"searches": 0, "nodes": 0, "lps": 0, "rounds": 0, "pivots": 0, "launches": 0}

    def extreme(which: str, order):
        """Rule 1: one LexicographicMIP() chain at gap 0 on the model loaded for its first objective; its point when
        it reached its end."""
        instance = solver._instance(jm[which], precision)  # loadJson only: no presolve
        tab = instance.tableau
        try:
            tab.setModel(instance)
            out = chain(tab, instance, jm[which], order, osenses, [0.0, 0.0], [0.0, 0.0], max_nodes, width, WHAT)
        except ValueError as e:  # the first level hit max_nodes before any integer plan
            raise ValueError(no_plan(keys[0 if which == "first" else 1], max_nodes)) from e
        finally:
            tab.close()
        count["searches"] += sum(1 for lv in out["levels"] if lv["kind"] is not None)
        for name in ("nodes", "lps", "rounds", "pivots", "launches"):
            count[name] += out[name]
        plan = None
        if out["stop"] == "reached":
            plan = point(instance, model, keys, senses, tuple(out["values"][v.id] for v in instance.variables))
        return out, plan

    ra, a = extreme("first", [o1, o2])
    if not ra["feasible"]:
        return dict(result(keys, senses, step, proven, [], None, None, 0.0), feasible=False, exact=True, **count)
    rb, b = extreme("second", [o2, o1])
    if not rb["feasible"]:
        raise RuntimeError(f"{WHAT}: the second objective's chain has no integer plan, but the first's found one")
    instance = solver._instance(jm["box"], precision)
    P = instance.precision
    stop = ends_stop(ra, rb)
    if stop is not None or same_image(a, b, P):
        return dict(result(keys, senses, step, proven, [a, b], None, stop or "reached", P), **count)

    slack, cost = box_edits(instance, model, keys, senses, (r1, r2))
    tab = instance.tableau
    try:
        tab.setModel(instance)
        tab.save()
        launches0 = tab.context.launches
        H, W = tab.height, tab.width
        n_ints = len(instance.initial_tableau().integerIndices)
        wave = iis.wave_width(tab.context, H + min(n_ints, 8), W)

        def stage(specs):
            edits = [node_spec(slack, cost, u1, u2, k) for u1, u2, k in specs]

            def evaluate(nodes):
                res = tab.box_batch([(edits[k], cuts) for k, cuts in nodes], check_cycles=True)
                count["pivots"] += int(res["pivots"].sum())
                return [node_of(res, i, H, cuts) for i, (_, cuts) in enumerate(nodes)]

            out = run(evaluate, [OWN] * len(specs), [math.inf] * len(specs), P, max_nodes, width, wave, shared=False)
            for name in ("nodes", "lps", "rounds"):
                count[name] += out[name]
            return [(state, None if w is None or state != "exact" else
                     point(instance, model, keys, senses, plan_of(instance, w)))
                    for state, w in zip(out["state"], out["witness"])]

        traced = trace(a, b, step, P, max_points, stage)
        count["launches"] += tab.context.launches - launches0
    finally:
        tab.close()
    count["searches"] += traced["searches"]
    return dict(result(keys, senses, step, proven, [a, b], traced, traced["stop"], P), **count)


def plan_of(instance, node) -> tuple:
    """The structural values of an integral node's final column 0, in instance.variables order."""
    at = plan_values(node.rhs, node.vrow)
    return tuple(at.get(v.index, 0.0) for v in instance.variables)

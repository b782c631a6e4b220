"""Multi-objective solving by compromise programming: mirror of the reference's `src/polyopt.ts`.

Each objective is optimized on its own (one `Solve` per objective, validate=True), the distinct optima are the
Pareto vertices, and a last `Solve` maximizes the sum of all variables subject to every objective sitting at the
average of its vertex values.  Returns {"midpoint", "vertices", "ranges"} (polyopt.ts:26-30).

`solver` needs only `Solve(model, precision, full, validate)`, like the reference's SolverLike.
"""
from __future__ import annotations

import json
import math
import random

from . import validation
from .model import _truthy, math_round, object_keys


def _is_number(v) -> bool:  # typeof v === "number"
    return isinstance(v, (int, float)) and not isinstance(v, bool)


def _js_num_str(x) -> str:
    """String(x) for a JavaScript number (integral values print without a fraction)."""
    if x != x:
        return "NaN"
    if x in (math.inf, -math.inf):
        return "Infinity" if x > 0 else "-Infinity"
    if float(x).is_integer() and abs(x) < 1e21:
        return str(int(x))
    return repr(float(x))


def _js_min(a, b):
    return math.nan if a != a or b != b else min(a, b)


def _js_max(a, b):
    return math.nan if a != a or b != b else max(a, b)


def _clone(model: dict) -> dict:
    """JSON.parse(JSON.stringify(model)) (polyopt.ts:36-38): non-finite numbers become null."""
    return json.loads(json.dumps(model), parse_constant=lambda _: None)


def _keys(obj) -> list:
    if isinstance(obj, dict):
        return object_keys(obj)
    if isinstance(obj, str):  # Object.keys of a string: its character indices
        return [str(i) for i in range(len(obj))]
    if obj is None:
        raise TypeError("Cannot convert undefined or null to object")
    return []


def _as_solution(value) -> dict:  # polyopt.ts:40-46
    if isinstance(value, dict):
        return value
    raise ValueError("Polyopt requires the solver to return an object result.")


def _backfill(solution: dict, model: dict, objective_keys: list) -> None:  # polyopt.ts:53-77
    variables = model["variables"]
    for attribute in objective_keys:
        if _truthy(variables.get(attribute)):  # an explicit variable keeps its own value
            continue
        if not _is_number(solution.get(attribute)):
            solution[attribute] = 0
        for name in object_keys(variables):
            contribution = variables[name].get(attribute)
            value = solution.get(name)
            if _is_number(contribution) and _is_number(value):
                solution[attribute] += value * contribution


def _vector_key(solution: dict, objective_keys: list) -> str:  # polyopt.ts:84-95
    parts = []
    for key in objective_keys:
        value = solution.get(key)
        parts.append(_js_num_str(math_round(value * 1000) / 1000) if _is_number(value) else "0")
    return "base-" + "-".join(parts)


def _ranges(vertices: list) -> dict:  # polyopt.ts:101-143
    ranges: dict = {}
    for vertex in vertices:
        for key in object_keys(vertex):
            value = vertex[key]
            if not _is_number(value):
                continue
            cur = ranges.get(key, {"min": math.inf, "max": -math.inf})
            ranges[key] = {"min": _js_min(cur["min"], value), "max": _js_max(cur["max"], value)}
    for vertex in vertices:
        for key in object_keys(ranges):
            if not _is_number(vertex.get(key)):
                vertex[key] = 0
            ranges[key]["min"] = _js_min(ranges[key]["min"], vertex[key])
            ranges[key]["max"] = _js_max(ranges[key]["max"], vertex[key])
    for key in object_keys(ranges):
        if not math.isfinite(ranges[key]["min"]):
            ranges[key] = {"min": 0, "max": 0}
    return ranges


def Polyopt(solver, model: dict) -> dict:  # polyopt.ts:150-223
    working = _clone(model)
    objectives = working.get("optimize")
    objective_keys = _keys(objectives)
    if len(objective_keys) == 0:
        raise ValueError("Multi-objective solve requires at least one objective definition.")
    working.pop("optimize", None)
    working.pop("opType", None)

    aggregated = {key: 0 for key in objective_keys}
    unique: set = set()
    vertices: list = []

    for name in objective_keys:  # polyopt.ts:172-199
        working["optimize"] = name
        working["opType"] = objectives[int(name)] if isinstance(objectives, str) else objectives[name]
        solution = _as_solution(solver.Solve(working, None, None, True))
        _backfill(solution, working, objective_keys)
        key = _vector_key(solution, objective_keys)
        if key in unique:
            continue
        unique.add(key)
        for k in objective_keys:
            value = solution.get(k)
            if _is_number(value):
                aggregated[k] += value
        vertices.append({k: v for k, v in solution.items() if k not in ("feasible", "result", "bounded")})

    for key in objective_keys:  # polyopt.ts:202-204
        working["constraints"][key] = {"equal": aggregated[key] / len(unique)}

    synthetic = "cheater-" + str(random.random())  # polyopt.ts:207-213
    working["optimize"] = synthetic
    working["opType"] = "max"
    for name in object_keys(working["variables"]):
        working["variables"][name][synthetic] = 1

    ranges = _ranges(vertices)
    midpoint = _as_solution(solver.Solve(working, None, None, True))
    return {"midpoint": midpoint, "vertices": vertices, "ranges": ranges}

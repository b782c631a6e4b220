"""Warm start of a continuous LP from a saved optimal basis.  DESIGN.md section 2f is the contract.

Solution.basis() exports the basis of a solved LP as JSON-serialisable names: the structural variables that are basic
and the rows whose slacks are non-basic (the binding rows).  Solve(model, basis=...) / Model.solve(basis=...) builds
and uploads the tableau as usual, crashes the named variables into it on the device (jslp_crash: each one pivots in on
the row with the largest |entry| among the rows the saved basis gives up) and then runs simplex() as usual.  The result
is an optimum of the same LP, shaped as Solve() shapes it; where the optimum is not unique it can be another optimal
vertex than the cold solve's.  This module checks the model and the basis, resolves the names (plan), and shapes the
crash records."""
from __future__ import annotations

import numpy as np

WHAT = "Solve(basis=...)"
REJECTED, BASIC = -1, -2  # record field 3 of jslp_crash when no pivot is done


def _name(con):
    return con.name if con.name is not None else con.index


def basis_of(m, vrow) -> dict:
    """The basis of model `m` whose tableau has the row labels `vrow`: {"variables": [id, ...], "constraints":
    [{"name": name, "type": "max" | "min"}, ...]}, structural basics in tableau row order, binding rows in row order."""
    by_index = {v.index: v for v in m.variables}
    basic = [int(x) for x in vrow[1:]]
    on_row = set(basic)
    variables = [by_index[x].id for x in basic if x in by_index]
    constraints = [{"name": _name(c), "type": "max" if c.isUpperBound else "min"}
                   for c in m.constraints if c.index not in on_row]
    return {"variables": variables, "constraints": constraints}


def basis(solution) -> dict:
    """Solution.basis(): the basis of the tableau as the solve of `solution` left it."""
    from .sensitivity import _check
    _check(solution, "basis()")
    t = solution._tableau
    return basis_of(t.model, t.varIndexByRow)


def _key(x):
    return not isinstance(x, bool) and isinstance(x, (str, int))


def _check_basis(b) -> None:
    if not isinstance(b, dict) or set(b) != {"variables", "constraints"}:
        raise ValueError(f"{WHAT}: a basis is a dict with exactly the keys 'variables' and 'constraints' "
                         "(Solution.basis() returns one)")
    if not isinstance(b["variables"], list) or not all(_key(v) for v in b["variables"]):
        raise ValueError(f"{WHAT}: basis['variables'] must be a list of variable ids")
    if not isinstance(b["constraints"], list):
        raise ValueError(f"{WHAT}: basis['constraints'] must be a list of {{'name': ..., 'type': 'max' | 'min'}}")
    for c in b["constraints"]:
        if not isinstance(c, dict) or set(c) != {"name", "type"} or not _key(c["name"]):
            raise ValueError(f"{WHAT}: a basis constraint is {{'name': ..., 'type': 'max' | 'min'}}, not {c!r}")
        if c["type"] not in ("max", "min"):
            raise ValueError(f"{WHAT}: a basis constraint's type is 'max' or 'min', not {c['type']!r}")


def plan(m, b) -> tuple:
    """(enter, leave, unknown) of basis `b` on model `m`, without a GPU: the structural labels to crash in, in basis
    order (int32); one byte per label, 1 where the saved basis gives up the label's row (the slacks of the named rows);
    and the names the model lacks, {"variables": [...], "constraints": [...]}."""
    _check_basis(b)
    var_of = {v.id: v for v in m.variables}
    rows: dict = {}
    for c in m.constraints:
        rows.setdefault((_name(c), "max" if c.isUpperBound else "min"), []).append(c)
    n_index = len(m.variables) + len(m.constraints)
    unknown = {"variables": [], "constraints": []}
    enter = []
    for vid in b["variables"]:
        if vid in var_of:
            enter.append(var_of[vid].index)
        else:
            unknown["variables"].append(vid)
    leave = np.zeros(n_index, dtype=np.uint8)
    for c in b["constraints"]:
        found = rows.get((c["name"], c["type"]))
        if found is None:
            unknown["constraints"].append(dict(c))
        for con in found or []:
            leave[con.index] = 1
    return np.asarray(enter, dtype=np.int32), leave, unknown


def check_model(m) -> None:
    """The refusals of a warm start that depend on the model alone."""
    if m.getNumberOfIntegerVariables() > 0:
        raise ValueError(f"{WHAT} is defined for continuous LPs only: the model has integer or binary variables")
    if any(c.relaxation is not None for c in m.constraints) or any(v.priority for v in m.variables):
        raise ValueError(f"{WHAT} does not support soft constraints (weight / priority) or optional objectives")
    if m.unrestrictedVariables:  # DESIGN.md section 7
        raise ValueError(f"{WHAT} does not support unrestricted variables: the simplex treats a variable it finds basic "
                         "as non-negative, so a crashed-in unrestricted variable can end on a wrong verdict")
    if m.tableauInitialized:
        raise ValueError(f"{WHAT} needs a model that has not been solved yet: its tableau already exists")


def report(m, records, n_pivots: int, unknown: dict) -> dict:
    """Solution.warmStart from the crash records (label, row, column, leaving label or REJECTED / BASIC)."""
    ids = {v.index: v.id for v in m.variables}
    out = {"pivots": int(n_pivots), "entered": [], "rejected": [], "alreadyBasic": [], "unknown": unknown}
    for rec in records:
        what = "alreadyBasic" if rec[3] == BASIC else "rejected" if rec[3] == REJECTED else "entered"
        out[what].append(ids[int(rec[0])])
    return out


def solve(m, b):
    """Model.solve(basis=b): presolve and upload as Model.solve() does, crash, simplex(), shape."""
    _check_basis(b)
    check_model(m)
    from .model import presolve
    if m.usePresolve and m.presolveResult is None:  # Model.solve (model.ts:427-449)
        m.presolveResult = presolve(m)
        if m.presolveResult.isInfeasible:
            m.tableau.model = m
            m.tableau.feasible = False
            sol = m.tableau.getSolution()
            sol.warmStart = None
            return sol
        for variable, value in m.presolveResult.fixedVariables.items():
            variable.value = value
            variable.cost = 0
    enter, leave, unknown = plan(m, b)
    t = m.tableau
    t.setModel(m)
    m.tableauInitialized = True
    records, n_pivots = t.crash(enter, leave)
    t.simplex()
    t.updateVariableValues()
    sol = t.getSolution()
    sol.warmStart = report(m, records, n_pivots, unknown)
    return sol

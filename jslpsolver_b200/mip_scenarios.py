"""What-if scenarios of a MIP: solve a model under many right-hand-side and cost edits in one call.  DESIGN.md section 2p
is the contract.

Result k is by definition Solve(edited_k): a deep copy of the JSON model with case k's values written into its
constraints' min / max / equal and its variables' objective coefficients, with options.presolve forced to False.  Such
an edit changes only column 0 and row 0 of the initial tableau, so the model is uploaded once and every scenario's
branch and cut runs side by side on the device (jslp_bnb_batch): each tree is jslp_branch_and_cut's default service,
committed in its own best-first order, and each round evaluates the open nodes of every live tree in shared launches.
Cases use the format of Solution.scenarios() (section 2e), which re-optimises warm from one solved LP under Model-API
semantics; Scenarios() cold-solves every edited model as Solve() would."""
from __future__ import annotations

import copy
import types
from typing import Any, Optional

import numpy as np

from . import validation
from .model import _truthy, object_keys
from .scenarios import _entries, edits_of
from .tableau import solution_set

WHAT = "Scenarios()"


def _refuse(model: dict, what: str = WHAT) -> None:
    """The model options Scenarios() (and TwoStage(), as `what`) refuse."""
    opt = model.get("optimize")
    if isinstance(opt, dict) and len(object_keys(opt)) > 1:
        raise ValueError(f"{what} takes one objective: `optimize` has {len(object_keys(opt))}")
    if model.get("external"):
        raise ValueError(f"{what} does not support external solvers")
    for spec in (model.get("constraints") or {}).values():
        if isinstance(spec, dict) and (spec.get("weight") is not None or spec.get("priority") is not None):
            raise ValueError(f"{what} does not support soft constraints (weight / priority)")
    options = model.get("options") or {}
    if _truthy(model.get("timeout")) or (_truthy(options) and _truthy(options.get("timeout"))):
        raise ValueError(f"{what} does not support timeout: a wall-clock stop cannot be reproduced when trees share "
                         "rounds")
    for key in ("useMIRCuts", "keep_solutions", "nodeSelection", "branching", "useIncremental"):
        if _truthy(options) and _truthy(options.get(key)):
            raise ValueError(f"{what} runs the default branch-and-cut service: options.{key} is not supported")


def _one_objective(model: dict) -> dict:
    """The model with a one-key `optimize` dict read as Solve() reads it: that key, maximised or minimised."""
    opt = model.get("optimize")
    if isinstance(opt, dict):
        key = object_keys(opt)[0]
        return dict(model, optimize=key, opType="max" if opt[key] == "max" else "min")
    return model


def edited(model: dict, m, spec) -> dict:
    """edited_k of DESIGN.md 2p: a deep copy of `model` with the values of `spec` written into it and presolve off.
    `m` is the base model as loadJson built it; the spec is checked as Solution.scenarios() checks it."""
    edits_of(m, spec, WHAT)
    out = copy.deepcopy(_one_objective(model))
    out["options"] = dict(out.get("options") or {}, presolve=False)
    cons = out["constraints"]
    for name, value in _entries(spec, "rhs", WHAT):
        c = cons[name]
        if isinstance(value, dict):
            if c.get("equal") is not None:
                raise ValueError(f"{WHAT}: constraint {name!r} is an equality: give one value")
            for side, v in value.items():
                c[side] = v
        elif c.get("equal") is not None:
            c["equal"] = value
        else:
            for side in ("min", "max"):
                if c.get(side) is not None:
                    c[side] = value
    objective = out.get("optimize")
    for vid, value in _entries(spec, "cost", WHAT):
        out["variables"][vid][objective] = value
    return out


def edges(base, it) -> tuple:
    """(column 0, row 0) of the initial tableau `it` of an edited model, checked bit for bit to differ from the base's
    `base` nowhere else; ValueError when the edit would solve a different model."""
    same = (it.matrix.shape == base.matrix.shape and np.array_equal(it.matrix[1:, 1:].view(np.uint64),
                                                                     base.matrix[1:, 1:].view(np.uint64))
            and np.array_equal(it.varIndexByRow, base.varIndexByRow)
            and np.array_equal(it.varIndexByCol, base.varIndexByCol)
            and np.array_equal(it.integerIndices, base.integerIndices)
            and np.array_equal(it.unrestricted, base.unrestricted))
    if not same:
        raise ValueError(f"{WHAT}: a case changes more than the right-hand sides and costs of the tableau")
    return it.matrix[:, 0].copy(), it.matrix[0, :].copy()


def Scenarios(solver, model: Any, cases, width=None, precision: Optional[float] = None, validate: bool = False) -> list:
    """See the module docstring.  `solver` supplies the engine settings of the tableau (Solver._instance); `width`
    tunes the speculation only."""
    from .model import Model
    from .pool import _count
    if validate:
        model = validation.validate(model)
    if not model:
        raise ValueError("Solver requires a model to operate on")
    if not isinstance(model, dict):
        raise ValueError(f"{WHAT} takes a JSON model")
    _refuse(model)
    if not isinstance(cases, (list, tuple)):
        raise ValueError(f"{WHAT} takes a list of scenarios, not {type(cases).__name__}")
    width = solver.max_spec_batch if width is None else _count("width", width, 1, WHAT)
    model = _one_objective(model)
    base_json = dict(model, options=dict(model.get("options") or {}, presolve=False))
    instance = solver._instance(base_json, precision)
    base = instance.initial_tableau()
    col0, row0 = [], []
    for spec in cases:  # every case is checked before anything runs
        it = Model(instance.precision).loadJson(edited(model, instance, spec)).initial_tableau()
        c, r = edges(base, it)
        col0.append(c)
        row0.append(r)
    if not cases:
        return []
    tab = instance.tableau
    try:
        tab.setModel(instance)
        out = tab.bnb_batch(np.array(col0), np.array(row0), tolerance=float(instance.tolerance or 0),
                            max_nodes=int(getattr(instance, "max_nodes", 0) or 0), width=width)
    finally:
        tab.close()
    from .solver import Solver
    results = []
    mip = instance.getNumberOfIntegerVariables() > 0
    for k, st in enumerate(out["status"]):
        h = int(out["height"][k])
        evaluation = st.evaluation if instance.isMinimization else -st.evaluation  # Tableau.getSolution
        sol = types.SimpleNamespace(feasible=bool(st.feasible), evaluation=evaluation, bounded=bool(st.bounded),
                                    _tableau=types.SimpleNamespace(isIntegralFlag=True if mip and st.is_integral
                                                                   else None))
        sol.solutionSet = solution_set(out["rhs"][k, :h], out["vrow"][k, :h], instance.precision,
                                       instance.variablesPerIndex)
        results.append(Solver._simplified(sol))
    return results

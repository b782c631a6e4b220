"""Pre-solve model checks: mirror of the reference's `src/validation.ts`, which `Solve(model, ..., validate=True)`
runs before it loads the model (main.ts:101-108).  Both functions take a JSON model, may mutate it in place as
the JavaScript does, and return it."""
from __future__ import annotations

import random
import warnings

from .model import _truthy, object_keys

PROPERTY_TYPOS = {  # validation.ts:14-32
    "optype": "opType", "OpType": "opType", "op_type": "opType", "type": "opType",
    "optimise": "optimize", "Optimize": "optimize", "objective": "optimize",
    "constraint": "constraints", "Constraints": "constraints",
    "variable": "variables", "Variables": "variables", "vars": "variables",
    "int": "ints", "integers": "ints", "Ints": "ints",
    "binary": "binaries", "Binaries": "binaries",
}

CONSTRAINT_TYPOS = {  # validation.ts:37-45
    "minimum": "min", "maximum": "max", "Min": "min", "Max": "max",
    "eq": "equal", "equals": "equal", "Equal": "equal",
}


def WarnOnTypos(model: dict) -> dict:  # validation.ts:53-100
    keys = object_keys(model)
    for key in keys:
        correction = PROPERTY_TYPOS.get(key)
        if correction:
            warnings.warn(f"[jsLPSolver] Warning: Model has '{key}' but expected '{correction}'. "
                          f"This may cause unexpected behavior.")
    if not _truthy(model.get("optimize")) and not any(PROPERTY_TYPOS.get(k) == "optimize" for k in keys):
        warnings.warn("[jsLPSolver] Warning: Model is missing 'optimize' property. "
                      "The solver needs to know which attribute to optimize.")
    if not _truthy(model.get("opType")) and not any(PROPERTY_TYPOS.get(k) == "opType" for k in keys):
        warnings.warn("[jsLPSolver] Warning: Model is missing 'opType' property. "
                      "Defaulting to 'max'. Use 'opType: \"max\"' or 'opType: \"min\"' to be explicit.")
    constraints = model.get("constraints")
    if _truthy(constraints) and isinstance(constraints, dict):
        for name in object_keys(constraints):
            constraint = constraints[name]
            if isinstance(constraint, dict):
                for prop in object_keys(constraint):
                    correction = CONSTRAINT_TYPOS.get(prop)
                    if correction:
                        warnings.warn(f"[jsLPSolver] Warning: Constraint '{name}' has '{prop}' "
                                      f"but expected '{correction}'.")
    return model


def _rename_attribute(model: dict, attribute: str) -> None:
    """validation.ts:116-126 / 137-146: the constraint named like the objective attribute moves to a random
    attribute name.  It is deleted and re-inserted, so it ends up LAST in the constraint order."""
    fake = str(random.random())
    variables = model["variables"]
    for x in object_keys(variables):
        if _truthy(variables[x].get(attribute)):
            variables[x][fake] = variables[x][attribute]
    constraints = model["constraints"]
    constraints[fake] = constraints[attribute]
    del constraints[attribute]


def CleanObjectiveAttributes(model: dict) -> dict:  # validation.ts:108-152
    optimize = model.get("optimize")
    if isinstance(optimize, str):
        if _truthy(model["constraints"].get(optimize)):
            _rename_attribute(model, optimize)
        return model
    if isinstance(optimize, dict):  # multi-objective: for-in over optimize, deleting only the current key
        for z in object_keys(optimize):
            constraint = model["constraints"].get(z)
            if _truthy(constraint):
                if constraint == "equal":  # an equality-constrained attribute cannot be optimized
                    del optimize[z]
                else:
                    _rename_attribute(model, z)
    return model


# `for (const test in validation)` (main.ts:102) walks the module namespace object, whose keys are sorted.
VALIDATORS = (CleanObjectiveAttributes, WarnOnTypos)


def validate(model: dict) -> dict:
    """What `Solve(model, ..., validate=true)` does to the model before loading it (main.ts:101-108)."""
    for validator in VALIDATORS:
        model = validator(model)
    return model

"""The contract of DESIGN.md section 2p restated literally over the C oracle: result k of Scenarios(model, cases) is the
oracle's Solve() (orc_branch_and_cut for a MIP, its simplex for a continuous LP, shaped as Solve() shapes a result) of
edited_k, the model with case k's values written in and presolve off.  No batching, no device."""
from __future__ import annotations

from jslpsolver_b200 import mip_scenarios as MS
from jslpsolver_b200.model import Model
from oracle import ref_model


def base_model(jm: dict) -> Model:
    """The base model as loadJson builds it, presolve off: what the case checks resolve names against."""
    return Model().loadJson(dict(MS._one_objective(jm), options={"presolve": False}))


def scenarios(jm: dict, cases: list) -> list:
    m = base_model(jm)
    return [ref_model.Solve(MS.edited(jm, m, spec)) for spec in cases]

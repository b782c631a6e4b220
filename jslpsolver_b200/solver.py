"""`solver.Solve(model)` -- mirror of the reference's public entry point (src/main.ts:94-193)
with the LP/MIP path running on the H100.  Same JSON model in, same result shape out."""
from __future__ import annotations

from typing import Any, Optional

from . import validation
from .conflict import Conflict as _conflict
from .frontier import Frontier as _frontier
from .frontier_mip import FrontierMIP as _frontier_mip
from .lexicographic import Lexicographic as _lexicographic
from .lexicographic_mip import LexicographicMIP as _lexicographic_mip
from .mip_scenarios import Scenarios as _scenarios
from .mip_variability import Variability as _variability
from .model import Model, object_keys
from .polyopt import Polyopt
from .pool import Pool as _pool
from .repair import Repair as _repair
from .repair_mip import RepairMIP as _repair_mip
from .two_stage import TwoStage as _two_stage


class Solver:
    Model = Model

    def __init__(self):
        self.lastSolvedModel: Optional[Model] = None
        self.engine = 0            # JSLP_OPT_ENGINE for every tableau this solver creates
        self.max_spec_batch = 0    # branch-and-cut speculation width (0 = library default)
        self.node_slots = None     # HBM-resident node batch width (None = auto, 0 = one node at a time)
        self.slot_steps = None
        self.options: dict = {}    # JSLP_OPT_* -> value for every tableau this solver creates (tuning / test aids)

    def Solve(self, model: Any, precision: Optional[float] = None, full: bool = False, validate: bool = False, *,
              basis: Optional[dict] = None, start=None, start_nodes: int = 1000):
        """main.ts Solve.  `basis` warm-starts a continuous LP (DESIGN.md section 2f); `start`, a {variable: value}
        plan or a list of them, seeds the branch and cut of a MIP with at most `start_nodes` node LPs per start to
        complete each (DESIGN.md section 2t), reported under Solution.mipStart with full=True."""
        if start is not None:
            return self._solve_start(model, precision, full, validate, basis, start, start_nodes)
        if basis is not None:  # warm start from a saved basis (DESIGN.md section 2f)
            return self._solve_warm(model, precision, full, validate, basis)
        if validate:
            model = validation.validate(model)  # main.ts:101-108
        if not model:
            raise ValueError("Solver requires a model to operate on")  # main.ts:110-112
        if isinstance(model, dict):
            opt = model.get("optimize")
            if isinstance(opt, dict) and len(opt) > 1:  # main.ts:115-119
                return Polyopt(self, model)
            if model.get("external"):
                raise NotImplementedError("external solvers (src/external) are out of scope")
        instance = self._instance(model, precision)
        solution = instance.solve()
        return self._finish(instance, solution, full)

    def _solve_warm(self, model: Any, precision: Optional[float], full: bool, validate: bool, basis: dict):
        from .warmstart import WHAT
        if validate:
            model = validation.validate(model)
        if not model:
            raise ValueError("Solver requires a model to operate on")
        if isinstance(model, dict):
            opt = model.get("optimize")
            if isinstance(opt, dict) and len(opt) > 1:
                raise ValueError(f"{WHAT} does not support multi-objective models (optimize with several objectives)")
            if model.get("external"):
                raise NotImplementedError("external solvers (src/external) are out of scope")
        instance = self._instance(model, precision)
        solution = instance.solve(basis=basis)
        return self._finish(instance, solution, full)

    def _solve_start(self, model: Any, precision: Optional[float], full: bool, validate: bool, basis, start,
                     start_nodes: int):
        from .mipstart import check_json
        if validate:
            model = validation.validate(model)
        if not model:
            raise ValueError("Solver requires a model to operate on")
        if isinstance(model, dict):
            check_json(model, basis)
        elif basis is not None:
            check_json({}, basis)
        instance = self._instance(model, precision)
        solution = instance.solve(start=start, start_nodes=start_nodes)
        return self._finish(instance, solution, full)

    def MultiObjective(self, model: dict):  # main.ts:209-211
        return Polyopt(self, model)

    def Frontier(self, model: dict, precision: Optional[float] = None, validate: bool = False) -> dict:
        """The Pareto frontier of a continuous LP with exactly two objectives: every efficient vertex from the first
        objective's optimum to the second's, with the weights that select it (frontier.py, DESIGN.md section 2g)."""
        return _frontier(self, model, precision, validate)

    def FrontierMIP(self, model: dict, *, step=None, max_points=1000, max_nodes=10000, width=None,
                    precision: Optional[float] = None, validate: bool = False) -> dict:
        """The Pareto frontier of a MIP with exactly two objectives: every nondominated image over the integer plans,
        from the first objective's lexicographic optimum to the second's, each box of the balanced box method searched
        exactly (frontier_mip.py, DESIGN.md section 2s).  `width` tunes the batching only."""
        return _frontier_mip(self, model, step=step, max_points=max_points, max_nodes=max_nodes, width=width,
                             precision=precision, validate=validate)

    def Lexicographic(self, model: dict, gap=0.0, absolute_gap=0.0, precision: Optional[float] = None,
                      validate: bool = False) -> dict:
        """Hierarchical objectives of a continuous LP: the objectives of `optimize` in order, each optimised over the
        plans within an allowance of every earlier optimum (lexicographic.py, DESIGN.md section 2j)."""
        return _lexicographic(self, model, gap, absolute_gap, precision, validate)

    def LexicographicMIP(self, model: dict, gap=0.0, absolute_gap=0.0, max_nodes=10000, width=None,
                         precision: Optional[float] = None, validate: bool = False) -> dict:
        """Hierarchical objectives of a MIP: the objectives of `optimize` in order, each optimised exactly over the
        integer plans within an allowance of every earlier optimum, one branch and bound per level
        (lexicographic_mip.py, DESIGN.md section 2q).  `width` tunes the batching only."""
        return _lexicographic_mip(self, model, gap, absolute_gap, max_nodes, width, precision, validate)

    def Repair(self, model: dict, weights=None, *, objective: bool = True, gap=0.0, absolute_gap=0.0,
               precision: Optional[float] = None, validate: bool = False) -> dict:
        """The least weighted relaxation of the rows of a (possibly infeasible) continuous LP, then its objective
        optimised over the plans that reach it (repair.py, DESIGN.md section 2k)."""
        return _repair(self, model, weights, objective=objective, gap=gap, absolute_gap=absolute_gap,
                       precision=precision, validate=validate)

    def RepairMIP(self, model: dict, weights=None, *, objective: bool = True, gap=0.0, absolute_gap=0.0,
                  max_nodes=10000, width=None, precision: Optional[float] = None, validate: bool = False) -> dict:
        """The least weighted relaxation of the rows of a (possibly infeasible) MIP over integer plans, then its
        objective optimised over the integer plans that reach it, each stage an exact branch and bound
        (repair_mip.py, DESIGN.md section 2r).  `width` tunes the batching only."""
        return _repair_mip(self, model, weights, objective=objective, gap=gap, absolute_gap=absolute_gap,
                           max_nodes=max_nodes, width=width, precision=precision, validate=validate)

    def Pool(self, model: dict, k=10, gap=0.0, absolute_gap=0.0, precision: Optional[float] = None,
             validate: bool = False, max_nodes=100000, width=None) -> dict:
        """The k best distinct integer assignments of a MIP, best first, each with its continuous completion, up to an
        allowance of the optimum (pool.py, DESIGN.md section 2m).  `width` tunes the speculation only."""
        return _pool(self, model, k, gap, absolute_gap, precision, validate, max_nodes, width)

    def Conflict(self, model: dict, max_nodes=10000, width=None, depth=None, precision: Optional[float] = None,
                 validate: bool = False) -> dict:
        """An irreducible set of rows and integrality restrictions of a MIP that has no integer plan, each member with
        the plan that breaks only it (conflict.py, DESIGN.md section 2n).  `width` / `depth` tune the batching only."""
        return _conflict(self, model, max_nodes, width, depth, precision, validate)

    def Variability(self, model: dict, gap=0.0, absolute_gap=0.0, variables=None, constraints=None, points=False,
                    max_nodes=10000, width=None, precision: Optional[float] = None, validate: bool = False) -> dict:
        """The range of every variable and slack of a MIP over all integer plans within an allowance of the optimum,
        each end exact or bounded (mip_variability.py, DESIGN.md section 2o).  `width` tunes the batching only."""
        return _variability(self, model, gap, absolute_gap, variables, constraints, points, max_nodes, width, precision,
                            validate)

    def Scenarios(self, model: dict, cases, *, width=None, precision: Optional[float] = None,
                  validate: bool = False) -> list:
        """What-if scenarios of a model: for each case {"rhs": {constraint: value or {"min", "max"}}, "cost": {variable:
        value}}, exactly Solve() of the model with those values written in and presolve off, every scenario's branch
        and cut run side by side on the device (mip_scenarios.py, DESIGN.md section 2p).  `width` tunes the batching
        only."""
        return _scenarios(self, model, cases, width, precision, validate)

    def TwoStage(self, model: dict, cases, first, probabilities=None, *, gap=1e-9, absolute_gap=None,
                 max_iterations=200, precision: Optional[float] = None, validate: bool = False) -> dict:
        """A two-stage stochastic LP: the first-stage plan over the variables `first` that minimises (or maximises)
        its cost plus the expected cost of each case's recourse plan, by the L-shaped method with every case's recourse
        LP batched on the device (two_stage.py, DESIGN.md section 2u).  Cases take "rhs" and "cost" of second-stage
        rows and variables as Scenarios() does, and "coefficients": {constraint: {first-stage variable: value}}."""
        return _two_stage(self, model, cases, first, probabilities, gap=gap, absolute_gap=absolute_gap,
                          max_iterations=max_iterations, precision=precision, validate=validate)

    def _instance(self, model: Any, precision: Optional[float]) -> Model:
        if isinstance(model, dict):
            options = model.get("options") or {}
            instance = Model(precision).loadJson(model)
            # selectBranchAndCutService (main.ts:62-83): incremental if explicitly asked, else enhanced if a strategy is named
            if options.get("useIncremental") is True or options.get("nodeSelection") or options.get("branching"):
                instance.branchAndCutOptions = {"nodeSelection": options.get("nodeSelection"), "branching": options.get("branching"),
                                                "useIncremental": options.get("useIncremental") is True}
        else:
            instance = model
        instance.tableau.engine = self.engine
        instance.tableau.max_spec_batch = self.max_spec_batch
        instance.tableau.node_slots = self.node_slots
        instance.tableau.slot_steps = self.slot_steps
        instance.tableau.options.update(self.options)
        return instance

    def _finish(self, instance: Model, solution, full: bool):  # main.ts:137-146
        self.lastSolvedModel = instance
        solution.solutionSet = solution.generateSolutionSet()
        if full:
            return solution
        return self._simplified(solution)

    @staticmethod
    def _simplified(solution) -> dict:  # main.ts:173-193
        head = {"feasible": solution.feasible, "result": solution.evaluation, "bounded": solution.bounded}
        if solution._tableau.isIntegralFlag:
            head["isIntegral"] = True
        values = {k: v for k, v in solution.solutionSet.items() if v != 0}
        out = {}
        keys = object_keys(values)
        for k in keys:  # JS objects list integer-like keys first
            if k.isdigit():
                out[k] = values[k]
        out.update(head)
        for k in keys:
            if not k.isdigit():
                out[k] = values[k]
        return out


solver = Solver()


def Solve(model: Any, precision: Optional[float] = None, full: bool = False, validate: bool = False, *,
          basis: Optional[dict] = None, start=None, start_nodes: int = 1000):
    return solver.Solve(model, precision, full, validate, basis=basis, start=start, start_nodes=start_nodes)


def Frontier(model: dict, precision: Optional[float] = None, validate: bool = False) -> dict:
    return solver.Frontier(model, precision, validate)


def FrontierMIP(model: dict, *, step=None, max_points=1000, max_nodes=10000, width=None,
                precision: Optional[float] = None, validate: bool = False) -> dict:
    return solver.FrontierMIP(model, step=step, max_points=max_points, max_nodes=max_nodes, width=width,
                              precision=precision, validate=validate)


def Lexicographic(model: dict, gap=0.0, absolute_gap=0.0, precision: Optional[float] = None,
                  validate: bool = False) -> dict:
    return solver.Lexicographic(model, gap, absolute_gap, precision, validate)


def LexicographicMIP(model: dict, gap=0.0, absolute_gap=0.0, max_nodes=10000, width=None,
                     precision: Optional[float] = None, validate: bool = False) -> dict:
    return solver.LexicographicMIP(model, gap, absolute_gap, max_nodes, width, precision, validate)


def Repair(model: dict, weights=None, *, objective: bool = True, gap=0.0, absolute_gap=0.0,
           precision: Optional[float] = None, validate: bool = False) -> dict:
    return solver.Repair(model, weights, objective=objective, gap=gap, absolute_gap=absolute_gap,
                         precision=precision, validate=validate)


def RepairMIP(model: dict, weights=None, *, objective: bool = True, gap=0.0, absolute_gap=0.0, max_nodes=10000,
              width=None, precision: Optional[float] = None, validate: bool = False) -> dict:
    return solver.RepairMIP(model, weights, objective=objective, gap=gap, absolute_gap=absolute_gap,
                            max_nodes=max_nodes, width=width, precision=precision, validate=validate)


def Pool(model: dict, k=10, gap=0.0, absolute_gap=0.0, precision: Optional[float] = None, validate: bool = False,
         max_nodes=100000, width=None) -> dict:
    return solver.Pool(model, k, gap, absolute_gap, precision, validate, max_nodes, width)


def Conflict(model: dict, max_nodes=10000, width=None, depth=None, precision: Optional[float] = None,
             validate: bool = False) -> dict:
    return solver.Conflict(model, max_nodes, width, depth, precision, validate)


def Scenarios(model: dict, cases, *, width=None, precision: Optional[float] = None, validate: bool = False) -> list:
    return solver.Scenarios(model, cases, width=width, precision=precision, validate=validate)


def TwoStage(model: dict, cases, first, probabilities=None, *, gap=1e-9, absolute_gap=None, max_iterations=200,
             precision: Optional[float] = None, validate: bool = False) -> dict:
    return solver.TwoStage(model, cases, first, probabilities, gap=gap, absolute_gap=absolute_gap,
                           max_iterations=max_iterations, precision=precision, validate=validate)


def Variability(model: dict, gap=0.0, absolute_gap=0.0, variables=None, constraints=None, points=False,
                max_nodes=10000, width=None, precision: Optional[float] = None, validate: bool = False) -> dict:
    return solver.Variability(model, gap, absolute_gap, variables, constraints, points, max_nodes, width, precision,
                              validate)

"""GpuTableau: the reference's `Tableau` seam (src/tableau/tableau.ts) with storage, pivot loop
and branch-and-cut on the H100 behind the C ABI (include/jslp_b200.h).

Method names, flags and read-back state follow the reference 1:1 (SURVEY.md 8b):
  simplex/phase1/phase2/pivot      tableau.ts:103-123   -> jslp_simplex/phase1/phase2/pivot
  save/restore                     tableau.ts:223-229   -> jslp_save/restore
  addCutConstraints / applyCuts    tableau.ts:145,240   -> jslp_add_cuts / jslp_apply_cuts
  isIntegral/getMostFractionalVar  tableau.ts:135,163   -> jslp_is_integral / jslp_most_fractional
  branchAndCut                     tableau.ts:244-246   -> jslp_branch_and_cut (or an injected service)
  solve/getSolution                tableau.ts:250-274
`matrix` is materialised lazily from the device (the authoritative copy lives in HBM).
There is no CPU path: every numerical method raises JslpError without the CUDA library + a GPU.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import numpy as np

from . import _lib
from ._lib import BnbOpts, BnbStatus, Cut, JslpError, LpStatus, ScenarioEdit, StartStatus

EPSILON = 2.220446049250313e-16

_CTX: dict[int, "DeviceContext"] = {}


class DeviceContext:
    """One jslp_ctx per GPU (launches on torch's current stream when torch is initialised)."""

    def __init__(self, device: int = 0, stream: Optional[int] = None):
        self.lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self.lib.jslp_ctx_create(device, C.c_void_p(stream) if stream else None, C.byref(h)))
        self.handle = h
        self.device = device

    @property
    def launches(self) -> int:
        return int(self.lib.jslp_ctx_launches(self.handle))

    def sync(self) -> None:
        _lib.check(self.lib.jslp_ctx_sync(self.handle))

    def close(self) -> None:
        if self.handle:
            self.lib.jslp_ctx_destroy(self.handle)
            self.handle = None


def default_context(device: Optional[int] = None) -> DeviceContext:
    import os
    if device is None:
        device = int(os.environ.get("JSLP_DEVICE", os.environ.get("LOCAL_RANK", "0")))
    if device not in _CTX:
        _CTX[device] = DeviceContext(device)
    return _CTX[device]


def js_round(x: float) -> float:
    if x != x or math.isinf(x):
        return x
    f = math.floor(x)
    return float(f + 1) if x - f >= 0.5 else float(f)


def solution_set(rhs, vrow, precision: float, variablesPerIndex: dict) -> dict:
    """generateSolutionSet (solution.ts:35-60) over a right-hand-side column and its row labels: every structural
    variable that is basic, rounded to the model precision."""
    out: dict = {}
    rounding = js_round(1 / precision)
    for r in range(1, len(vrow)):
        var = variablesPerIndex.get(int(vrow[r]))
        if var is None or var.isSlack:
            continue
        out[var.id] = js_round((EPSILON + float(rhs[r])) * rounding) / rounding
    return out


class Solution:  # solution.ts:16-61
    def __init__(self, tableau: "GpuTableau", evaluation: float, feasible: bool, bounded: bool):
        self.feasible, self.evaluation, self.bounded = feasible, evaluation, bounded
        self._tableau = tableau
        self._version = getattr(tableau, "_version", None)  # the tableau state this solution describes
        self.solutionSet: dict = {}

    warmStart = None  # Solve(model, full=True, basis=...): what the crash did (DESIGN.md section 2f)

    def basis(self) -> dict:
        """The basis of this continuous LP optimum as JSON-serialisable names, {"variables": [basic variable ids],
        "constraints": [{"name", "type"} of the binding rows]}, for Solve(model, basis=...) (DESIGN.md section 2f);
        raises ValueError where sensitivity() does."""
        from .warmstart import basis
        return basis(self)

    def sensitivity(self) -> dict:
        """Shadow prices, reduced costs and right-hand-side / cost ranges of this continuous LP optimum
        (DESIGN.md section 2b); raises ValueError where they are not defined."""
        from .sensitivity import report
        return report(self)

    def iis(self) -> dict:
        """An irreducible infeasible subset of the rows of this infeasible continuous LP (DESIGN.md section 2c):
        {"constraints": [{name, type, rhs}, ...], "names": [...], "irreducible": bool, "lps": int}; raises
        ValueError where it is not defined."""
        from .iis import compute
        return compute(self)

    def unbounded(self, width=None) -> dict:
        """Why this continuous LP is unbounded (DESIGN.md section 2l): the improving ray where the simplex stopped,
        {"ray", "rate", "point", "constraints", "blocking"}, whether a recession-cone LP confirms an improving direction
        ("confirmed"), an irreducible set of variables whose caps make the LP bounded ("bound": {"variables",
        "irreducible"}, None when undecided) and the cone LPs solved ("lps").  The tableau and the model are left
        unchanged; raises ValueError where it is not defined.  `width` tunes the schedule only."""
        from .unbounded import compute
        return compute(self, width=width)

    def parametric(self, constraint=None, variable=None, side=None, to=None) -> dict:
        """The optimal result of this continuous LP as one right-hand side (constraint=name, side= for a constraint
        with a min and a max bound) or one cost (variable=id) moves from its current value to `to`: linear pieces
        between the basis changes, each with its slope and the basis change that ends it (DESIGN.md section 2d).
        The tableau is left unchanged; raises ValueError where sensitivity() does and for unknown names."""
        from .parametric import compute
        return compute(self, constraint=constraint, variable=variable, side=side, to=to)

    def scenarios(self, cases) -> list:
        """What-if re-optimisation of this continuous LP: for each case {"rhs": {constraint: value, ...}, "cost":
        {variable: value, ...}}, the Solve() result of the model with those right-hand sides and costs, as
        Constraint.setRightHandSide / Model.setCost followed by a re-solve from this optimum would return it (DESIGN.md
        section 2e).  A constraint with a min and a max bound takes {"min": a, "max": b}.  The tableau and the model are
        left unchanged; raises ValueError where sensitivity() does, for unknown names and for bad values."""
        from .scenarios import compute
        return compute(self, cases)

    def variability(self, variables=None, constraints=None, points=False, *, gap=0.0, absolute_gap=0.0) -> dict:
        """Alternative optima of this continuous LP (DESIGN.md section 2h): over all optimal solutions, the range of
        every structural variable, {"value", "min", "max", "fixed"} under "variables", and of every row's slack,
        {"name", "type", "slack": {"value", "min", "max"}} under "constraints" in tableau order (an equality or a
        min+max constraint is two rows).  Ends are raw doubles, +-inf where the optimal face is unbounded, None where
        the LP behind an end gave no answer ("exact" is then False).  "unique" says whether every structural variable
        of the model moves by no more than the precision; it covers all of them even when variables= (a list of ids)
        or constraints= (a list of names) restricts what is reported.  points=True adds "argmin" / "argmax", the
        optimal vertex {id: value} where each end is reached.  "free" counts the non-basic columns at reduced cost 0,
        "lps" the LPs solved.  The tableau and the model are left unchanged; raises ValueError where sensitivity()
        does, for unknown names and for models with unrestricted variables.

        Near-optimal variability (DESIGN.md section 2i): with an allowance t = max(absolute_gap, gap * |result|) > 0,
        the ranges are taken over every feasible plan whose objective is at most t worse than the optimum instead, no
        column is banned ("free" counts every non-basic column), and the report gains "allowance": t.  t == 0, the
        default, is exactly the report above.  gap= and absolute_gap= must be finite numbers >= 0."""
        from .variability import compute
        return compute(self, variables=variables, constraints=constraints, points=points, gap=gap,
                       absolute_gap=absolute_gap)

    def generateSolutionSet(self) -> dict:
        t = self._tableau
        if t.handle is None:
            return {}
        return solution_set(t.rhs_column(), t.varIndexByRow, t.precision, t.variablesPerIndex)


class MilpSolution(Solution):  # solution.ts:66-80
    def __init__(self, tableau, evaluation, feasible, bounded, branchAndCutIterations):
        super().__init__(tableau, evaluation, feasible, bounded)
        self.iter = branchAndCutIterations


class GpuTableau:
    def __init__(self, precision: float = 1e-8, branchAndCutService=None, context: Optional[DeviceContext] = None):
        self.precision = precision
        self.branchAndCutService = branchAndCutService
        self.context = context
        self.model = None
        self.handle = None
        self.width = self.height = 0
        self.feasible = True
        self.bounded = True
        self.evaluation = 0.0
        self.bestPossibleEval = 0.0
        self.simplexIters = 0
        self.unboundedVarIndex = None
        self.branchAndCutIterations = 0
        self.__isIntegral = None
        self.nVars = 0
        self.lastElementIndex = 0
        self.variablesPerIndex: dict = {}
        self.optionalPriorities: list = []
        self.lastStatus: Optional[LpStatus] = None
        self.lastBnbStatus: Optional[BnbStatus] = None
        self.bestCuts: list = []
        self.engine = 0
        self.max_spec_batch = 0
        self.distributed = False  # True: branchAndCut shards node rounds over torch.distributed ranks
        self.shard_policy = 0     # jslp_bnb_opts.shard_policy: 0 = shard only rounds whose node LPs run in HBM, 1 = always
        self.node_slots = None    # JSLP_OPT_NODE_SLOTS (None = library default: auto)
        self.slot_steps = None    # JSLP_OPT_SLOT_STEPS
        self.options: dict = {}   # JSLP_OPT_* -> value, applied after every upload (tuning aids)
        self.availableIndexes: list = []   # tableau.ts:77
        self._cache: dict = {}
        self._cache_log = None
        self._version = 0          # bumped by every change of the device tableau (solves and edits)
        self._solved_version = -1  # _version right after the last simplex()

    # name-mangling-free accessor used by Solve (main.ts:180)
    @property
    def isIntegralFlag(self):
        return self.__isIntegral

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def close(self) -> None:
        if self.handle is not None and self.context is not None and self.context.handle:
            self.context.lib.jslp_tab_destroy(self.handle)
        self.handle = None

    # ------------------------------------------------------------------ setup
    def upload(self, matrix, varIndexByRow, varIndexByCol, unrestricted=None, integerIndices=None,
               optionalCosts=None, row_capacity: Optional[int] = None) -> "GpuTableau":
        """Tableau.initialize + _resetMatrix result -> device (tableau.ts:292-380)."""
        if self.context is None:
            self.context = default_context()
        L = self.context.lib
        M = np.ascontiguousarray(matrix, dtype=np.float64)
        H, W = M.shape
        self.close()
        h = C.c_void_p()
        cap = row_capacity if row_capacity else H + 64
        _lib.check(L.jslp_tab_create(self.context.handle, W, H, cap, float(self.precision), C.byref(h)))
        self.handle = h
        vrow = np.ascontiguousarray(varIndexByRow, dtype=np.int32)
        vcol = np.ascontiguousarray(varIndexByCol, dtype=np.int32)
        n_index = W + H - 2
        unres = None
        if unrestricted is not None and len(unrestricted):
            unres = np.zeros(n_index, dtype=np.uint8)
            unres[:len(unrestricted)] = np.asarray(unrestricted, dtype=np.uint8)[:n_index]
        ints = None if integerIndices is None else np.ascontiguousarray(integerIndices, dtype=np.int32)
        opt = None if optionalCosts is None or len(optionalCosts) == 0 else np.ascontiguousarray(optionalCosts, dtype=np.float64)
        self.nOpt = 0 if opt is None else opt.shape[0]
        _lib.check(L.jslp_tab_upload(
            self.handle, M.ctypes.data, vrow.ctypes.data, vcol.ctypes.data,
            None if unres is None else unres.ctypes.data, n_index,
            None if ints is None or len(ints) == 0 else ints.ctypes.data, 0 if ints is None else len(ints),
            self.nOpt, None if opt is None else opt.ctypes.data))
        self.width, self.height = W, H
        self.nVars = n_index
        self.lastElementIndex = n_index
        self.nInts = 0 if ints is None else len(ints)
        if self.engine:
            self.set_option(_lib.OPT_ENGINE, self.engine)
        for k, v in self.options.items():
            self.set_option(k, v)
        self._edited()
        self._cache_log = None
        return self

    def setModel(self, model) -> "GpuTableau":  # tableau.ts:382-391
        self.model = model
        it = model.initial_tableau()
        self.variablesPerIndex = model.variablesPerIndex
        self.optionalPriorities = it.optionalPriorities
        return self.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, it.integerIndices,
                           it.optionalCosts)

    def set_option(self, key: int, value: float) -> None:
        _lib.check(self.context.lib.jslp_tab_set_option(self._h(), key, float(value)))

    def _edited(self) -> None:
        self._cache.clear()
        self._version += 1

    def _h(self):
        if self.handle is None:
            raise JslpError("tableau has no device state: call setModel()/upload() first")
        return self.handle

    def _check_cycles(self) -> int:
        return int(bool(getattr(self.model, "checkForCycles", True)))

    def _absorb(self, st: LpStatus) -> None:
        self.lastStatus = st
        self.feasible = bool(st.feasible)
        self.bounded = bool(st.bounded)
        self.evaluation = st.evaluation
        self.bestPossibleEval = st.best_possible_eval
        self.simplexIters = st.simplex_iters
        self.unboundedVarIndex = None if st.unbounded_var_index < 0 else st.unbounded_var_index
        self.width, self.height = st.width, st.height
        if st.cycled and self.model is not None:  # simplex.ts:86-88 / 313-315
            self.model.messages += [f"Cycle in phase {st.cycled}", f"Start :{st.cycle_start}",
                                    f"Length :{st.cycle_length}"]
        self._edited()

    # ------------------------------------------------------------------ simplex (tableau.ts:103-123)
    def simplex(self, check_cycles: Optional[bool] = None) -> "GpuTableau":
        """jslp_simplex with the model's cycle check, unless check_cycles is given."""
        st = LpStatus()
        cc = self._check_cycles() if check_cycles is None else int(bool(check_cycles))
        _lib.check(self.context.lib.jslp_simplex(self._h(), cc, C.byref(st)))
        self._absorb(st)
        self._solved_version = self._version
        return self

    def phase1(self) -> int:
        st = LpStatus()
        _lib.check(self.context.lib.jslp_phase1(self._h(), self._check_cycles(), C.byref(st)))
        self._absorb(st)
        return st.phase1_pivots

    def phase2(self) -> int:
        st = LpStatus()
        _lib.check(self.context.lib.jslp_phase2(self._h(), self._check_cycles(), C.byref(st)))
        self._absorb(st)
        return st.phase2_pivots

    def pivot(self, pivotRowIndex: int, pivotColumnIndex: int) -> None:
        _lib.check(self.context.lib.jslp_pivot(self._h(), pivotRowIndex, pivotColumnIndex))
        self._edited()

    # ------------------------------------------------------------------ backup (tableau.ts:219-229)
    def save(self) -> None:
        _lib.check(self.context.lib.jslp_save(self._h()))

    def restore(self) -> None:
        _lib.check(self.context.lib.jslp_restore(self._h()))
        self._refresh_dims()

    def _refresh_dims(self) -> None:
        info = (C.c_int32 * 6)()
        _lib.check(self.context.lib.jslp_tab_info(self._h(), info))
        self.width, self.height, self.nVars, self.lastElementIndex = info[0], info[1], info[2], info[3]
        self._edited()

    def getNewElementIndex(self) -> int:  # tableau.ts:393-401
        if self.availableIndexes:
            return self.availableIndexes.pop()
        self._refresh_dims()
        index = self.lastElementIndex
        self.lastElementIndex += 1
        return index

    # ------------------------------------------------------------------ dynamic modification (dynamic-modification.ts)
    def _opt_slot(self, priority) -> int:
        if not priority:
            return -1
        if priority not in self.optionalPriorities:
            raise JslpError("an optional objective with a new priority needs setModel() again (the uploaded set is fixed)")
        return self.optionalPriorities.index(priority)

    def putInBase(self, varIndex: int) -> int:
        r = C.c_int()
        _lib.check(self.context.lib.jslp_put_in_base(self._h(), int(varIndex), C.byref(r)))
        self._edited()
        return r.value

    def takeOutOfBase(self, varIndex: int) -> int:
        c = C.c_int()
        _lib.check(self.context.lib.jslp_take_out_of_base(self._h(), int(varIndex), C.byref(c)))
        self._edited()
        return c.value

    def updateRightHandSide(self, constraint, difference: float) -> None:
        idx = constraint if isinstance(constraint, int) else constraint.index
        _lib.check(self.context.lib.jslp_update_rhs(self._h(), int(idx), float(difference)))
        self._edited()

    def updateConstraintCoefficient(self, constraint, variable, difference: float) -> None:
        ci = constraint if isinstance(constraint, int) else constraint.index
        vi = variable if isinstance(variable, int) else variable.index
        if ci == vi:  # dynamic-modification.ts:114-118
            raise ValueError("[Tableau.updateConstraintCoefficient] constraint index should not be equal to variable index !")
        _lib.check(self.context.lib.jslp_update_coefficient(self._h(), int(ci), int(vi), float(difference)))
        self._edited()

    def updateCost(self, variable, difference: float, priority: int = 0) -> None:
        vi = variable if isinstance(variable, int) else variable.index
        pr = priority if isinstance(variable, int) else variable.priority
        _lib.check(self.context.lib.jslp_update_cost(self._h(), int(vi), self._opt_slot(pr), float(difference)))
        self._edited()

    def addConstraint(self, constraint=None, *, isUpperBound=None, rhs=None, index=None, terms=None) -> None:
        if constraint is not None:
            isUpperBound, rhs, index = constraint.isUpperBound, constraint.rhs, constraint.index
            terms = [(t.variable.index, t.coefficient) for t in constraint.terms]
        terms = terms or []
        tv = np.ascontiguousarray([v for v, _ in terms], dtype=np.int32)
        tc = np.ascontiguousarray([c for _, c in terms], dtype=np.float64)
        _lib.check(self.context.lib.jslp_add_constraint(self._h(), int(bool(isUpperBound)), float(rhs), int(index),
                                                        tv.ctypes.data if len(terms) else None,
                                                        tc.ctypes.data if len(terms) else None, len(terms)))
        self._refresh_dims()

    def removeConstraint(self, constraint) -> None:
        idx = constraint if isinstance(constraint, int) else constraint.index
        _lib.check(self.context.lib.jslp_remove_constraint(self._h(), int(idx)))
        self.availableIndexes.append(idx)          # dynamic-modification.ts:246
        if not isinstance(constraint, int):
            constraint.slack.index = -1            # :248
        self._refresh_dims()

    def addVariable(self, variable=None, *, index=None, cost=0.0, priority=0, isInteger=False, isUnrestricted=False) -> None:
        if variable is not None:
            index, cost, priority, isInteger = variable.index, variable.cost, variable.priority, variable.isInteger
            isUnrestricted = bool(self.model is not None and self.model.unrestrictedVariables.get(index))
        is_min = True if self.model is None else self.model.isMinimization
        entry = -cost if is_min else cost                      # dynamic-modification.ts:258
        _lib.check(self.context.lib.jslp_add_variable(self._h(), int(index), float(entry), self._opt_slot(priority),
                                                      int(bool(isInteger)), int(bool(isUnrestricted))))
        self._refresh_dims()

    def removeVariable(self, variable) -> None:
        idx = variable if isinstance(variable, int) else variable.index
        _lib.check(self.context.lib.jslp_remove_variable(self._h(), int(idx)))
        self.availableIndexes.append(idx)          # dynamic-modification.ts:313
        self._refresh_dims()

    # ------------------------------------------------------------------ cuts / MIP helpers
    @staticmethod
    def _cut_array(cuts):
        arr = (Cut * max(1, len(cuts)))()
        for i, c in enumerate(cuts):
            if isinstance(c, dict):
                ty, vi, val = c["type"], c["varIndex"], c["value"]
            else:
                ty, vi, val = c
            arr[i].type = 0 if ty in (0, "min") else 1
            arr[i].var_index = int(vi)
            arr[i].value = float(val)
        return arr

    def addCutConstraints(self, branchingCuts) -> None:
        _lib.check(self.context.lib.jslp_add_cuts(self._h(), self._cut_array(branchingCuts), len(branchingCuts)))
        self._refresh_dims()

    def addLowerBoundMIRCut(self, rowIndex: int) -> bool:   # cutting-strategies.ts:74-134
        a = C.c_int()
        _lib.check(self.context.lib.jslp_add_mir_cut(self._h(), int(rowIndex), 0, C.byref(a)))
        self._refresh_dims()
        return bool(a.value)

    def addUpperBoundMIRCut(self, rowIndex: int) -> bool:   # cutting-strategies.ts:136-196
        a = C.c_int()
        _lib.check(self.context.lib.jslp_add_mir_cut(self._h(), int(rowIndex), 1, C.byref(a)))
        self._refresh_dims()
        return bool(a.value)

    def applyMIRCuts(self) -> None:                         # cutting-strategies.ts:198-212
        n = C.c_int()
        _lib.check(self.context.lib.jslp_apply_mir_cuts(self._h(), C.byref(n)))
        self._refresh_dims()

    def computeFractionalVolume(self, ignoreIntegerValues: bool = False) -> float:  # mip-utils.ts:67-98
        v = C.c_double()
        _lib.check(self.context.lib.jslp_fractional_volume(self._h(), int(bool(ignoreIntegerValues)), C.byref(v)))
        return v.value

    def _sync_mir_option(self) -> None:
        self.set_option(_lib.OPT_USE_MIR_CUTS, 1 if getattr(self.model, "useMIRCuts", False) else 0)

    def applyCuts(self, branchingCuts) -> None:
        if self.branchAndCutService is not None:
            self.branchAndCutService.applyCuts(self, branchingCuts)
            return
        self._sync_mir_option()
        st = LpStatus()
        _lib.check(self.context.lib.jslp_apply_cuts(self._h(), self._cut_array(branchingCuts), len(branchingCuts),
                                                    self._check_cycles(), C.byref(st)))
        self._absorb(st)

    def isIntegral(self) -> bool:
        v = C.c_int()
        _lib.check(self.context.lib.jslp_is_integral(self._h(), C.byref(v)))
        return bool(v.value)

    def getMostFractionalVar(self) -> dict:
        i, v = C.c_int32(), C.c_double()
        _lib.check(self.context.lib.jslp_most_fractional(self._h(), C.byref(i), C.byref(v)))
        return {"index": None if i.value < 0 else i.value, "value": v.value}

    def branchAndCut(self, start=None, start_nodes: int = 1000) -> None:  # tableau.ts:244-246
        """Branch and cut of the tableau; `start` (DESIGN.md section 2t) is a list of MIP starts, each a list of
        (type, varIndex, value) cuts on integer labels, seeding the incumbent through jslp_branch_and_cut_start, with
        at most `start_nodes` node LPs per start.  Their outcomes go to lastStartStatus."""
        if self.branchAndCutService is not None:
            self.branchAndCutService.branchAndCut(self)
            return
        m = self.model
        self._sync_mir_option()
        opts = BnbOpts()
        opts.tolerance = float(getattr(m, "tolerance", 0) or 0)
        opts.is_minimization = int(bool(getattr(m, "isMinimization", True)))
        opts.check_cycles = self._check_cycles()
        opts.max_spec_batch = int(self.max_spec_batch)
        opts.rank, opts.n_ranks = 0, 1
        keep = None
        if self.distributed:  # shard each round's nodes over ranks (one process per GPU)
            from . import distributed as D
            if D.is_active():
                opts.rank, opts.n_ranks = D.rank_and_world()
                comm = D.nccl_communicator(self.context)  # in-library NCCL; None under gloo (CPU tests, shared GPU)
                if comm is not None:
                    opts.comm = comm
                else:
                    opts.all_gather, keep = D.make_all_gather_hook()
        opts.shard_policy = int(self.shard_policy)
        sel = getattr(m, "branchAndCutOptions", None)  # main.ts:62-83: options.nodeSelection / options.branching
        if sel:
            opts.service = 2 if sel.get("useIncremental") else 1
            opts.node_selection = {"best-first": 1, "depth-first": 2, "hybrid": 3}[sel.get("nodeSelection") or "hybrid"]
            opts.branching = {"most-fractional": 1, "pseudocost": 2, "strong": 3}[sel.get("branching") or "pseudocost"]
        opts.max_nodes = int(getattr(m, "max_nodes", 0) or 0)
        # model.timeout [ms] and options.keep_solutions (model.ts:338-374; branch-and-cut.ts:61-63,76,143-153)
        opts.timeout_ms = float(getattr(m, "timeout", 0) or 0)
        opts.keep_solutions = int(bool(getattr(m, "keep_solutions", False)))
        if self.node_slots is not None:
            self.set_option(_lib.OPT_NODE_SLOTS, self.node_slots)
        if self.slot_steps is not None:
            self.set_option(_lib.OPT_SLOT_STEPS, self.slot_steps)
        st = BnbStatus()
        # a cut list holds at most one min and one max cut per integer variable
        cap = max(4096, 2 * getattr(self, "nInts", 0))
        best = (Cut * cap)()
        if start is None:
            _lib.check(self.context.lib.jslp_branch_and_cut(self._h(), C.byref(opts), C.byref(st), best, cap))
        else:
            offsets = np.zeros(len(start) + 1, dtype=np.int32)
            offsets[1:] = np.cumsum([len(c) for c in start])
            cuts = self._cut_array([c for cl in start for c in cl])
            status = (StartStatus * max(1, len(start)))()
            _lib.check(self.context.lib.jslp_branch_and_cut_start(self._h(), C.byref(opts), cuts, offsets.ctypes.data,
                                                                  len(start), int(start_nodes), status, C.byref(st),
                                                                  best, cap))
            self.lastStartStatus = [status[i] for i in range(len(start))]
        self.lastBnbStatus = st
        self.feasible, self.bounded = bool(st.feasible), bool(st.bounded)
        self.evaluation, self.bestPossibleEval = st.evaluation, st.best_possible_eval
        self.branchAndCutIterations = st.iterations
        if st.is_integral:
            self.__isIntegral = True
        self.bestCuts = [(best[i].type, best[i].var_index, best[i].value) for i in range(min(cap, st.n_best_cuts))]
        self._refresh_dims()
        if opts.keep_solutions and m is not None:  # branch-and-cut.ts:143-153
            for i in range(st.n_solutions):
                m.solutions = (m.solutions or []) + [self._stored_solution(i)]

    def _stored_solution(self, i: int) -> dict:
        """model.solutions[i]: generateSolutionSet() of incumbent i plus `result` (branch-and-cut.ts:144-152)."""
        L = self.context.lib
        ev, h = C.c_double(), C.c_int32()
        _lib.check(L.jslp_bnb_solution(self._h(), i, C.byref(ev), C.byref(h), None, None, 0))
        vrow, rhs = np.empty(h.value, dtype=np.int32), np.empty(h.value, dtype=np.float64)
        _lib.check(L.jslp_bnb_solution(self._h(), i, None, None, vrow.ctypes.data, rhs.ctypes.data, h.value))
        rounding = js_round(1 / self.precision)
        store: dict = {}
        for r in range(1, h.value):
            var = self.variablesPerIndex.get(int(vrow[r]))
            if var is None or var.isSlack:
                continue
            store[var.id] = js_round((EPSILON + float(rhs[r])) * rounding) / rounding
        is_min = True if self.model is None else self.model.isMinimization
        store["result"] = ev.value if is_min else -ev.value
        return store

    def bnb_batch(self, col0, row0, tolerance: float = 0.0, max_nodes: int = 0, width: int = 0,
                  check_cycles: Optional[bool] = None) -> dict:
        """jslp_bnb_batch: branch and cut (the default service) of this tableau with rows 1.. of column 0 replaced by
        col0[s] and row 0 by row0[s], for every scenario s (DESIGN.md section 2p); the root LP alone without integer
        variables.  Returns the per-scenario BnbStatus list, the final column 0 and row labels (rhs / vrow, n x
        row_stride, `height` entries each) and the kernel launches of the call.  The tableau, its snapshot and its
        scalar state are left as they were."""
        c0 = np.ascontiguousarray(col0, dtype=np.float64)
        r0 = np.ascontiguousarray(row0, dtype=np.float64)
        n = c0.shape[0]
        if n and (c0.shape[1] != self.height or r0.shape != (n, self.width)):
            raise ValueError(f"bnb_batch: column 0 / row 0 must be n x {self.height} / n x {self.width}")
        m = self.model
        opts = BnbOpts()
        opts.tolerance = float(tolerance)
        opts.is_minimization = int(bool(getattr(m, "isMinimization", True)))
        opts.check_cycles = self._check_cycles() if check_cycles is None else int(bool(check_cycles))
        opts.max_spec_batch = int(width)
        opts.rank, opts.n_ranks = 0, 1
        opts.max_nodes = int(max_nodes)
        stride = self.height + 2 * getattr(self, "nInts", 0)
        status = (BnbStatus * max(1, n))()
        rhs, vrow = np.zeros((n, stride), dtype=np.float64), np.zeros((n, stride), dtype=np.int32)
        height = np.zeros(n, dtype=np.int32)
        _lib.check(self.context.lib.jslp_bnb_batch(self._h(), c0.ctypes.data, r0.ctypes.data, n, C.byref(opts), stride,
                                                   status, rhs.ctypes.data, vrow.ctypes.data, height.ctypes.data))
        return {"status": [status[i] for i in range(n)], "rhs": rhs, "vrow": vrow, "height": height,
                "launches": int(status[0].kernel_launches) if n else 0}

    def node_log(self) -> np.ndarray:
        n = C.c_int64()
        L = self.context.lib
        _lib.check(L.jslp_bnb_node_log(self._h(), None, 0, C.byref(n)))
        out = np.empty((n.value, 8), dtype=np.float64)
        if n.value:
            _lib.check(L.jslp_bnb_node_log(self._h(), out.ctypes.data, n.value, C.byref(n)))
        return out

    # ------------------------------------------------------------------ read-back
    def _download(self, what: str):
        if what in self._cache:
            return self._cache[what]
        L = self.context.lib
        H, W = self.height, self.width
        if what == "matrix":
            out = np.empty((H, W), dtype=np.float64)
            _lib.check(L.jslp_download(self._h(), out.ctypes.data, None, None, None, None, None, None, None))
        elif what == "rhs":
            out = np.empty(H, dtype=np.float64)
            _lib.check(L.jslp_download(self._h(), None, out.ctypes.data, None, None, None, None, None, None))
        elif what == "cost":
            out = np.empty(W, dtype=np.float64)
            _lib.check(L.jslp_download(self._h(), None, None, out.ctypes.data, None, None, None, None, None))
        elif what == "maps":
            vr, vc = np.empty(H, dtype=np.int32), np.empty(W, dtype=np.int32)
            _lib.check(L.jslp_download(self._h(), None, None, None, vr.ctypes.data, vc.ctypes.data, None, None, None))
            out = (vr, vc)
        elif what == "opt":
            out = np.empty((self.nOpt, W), dtype=np.float64)
            if self.nOpt:
                _lib.check(L.jslp_download(self._h(), None, None, None, None, None, out.ctypes.data, None, None))
        else:
            raise KeyError(what)
        self._cache[what] = out
        return out

    @property
    def matrix(self) -> np.ndarray:
        """Flat row-major Float64Array view, stride == width (tableau.ts:49,304)."""
        return self._download("matrix").reshape(-1)

    def matrix2d(self) -> np.ndarray:
        return self._download("matrix")

    def rhs_column(self) -> np.ndarray:
        return self._download("rhs")

    def cost_row(self) -> np.ndarray:
        return self._download("cost")

    @property
    def varIndexByRow(self) -> np.ndarray:
        return self._download("maps")[0]

    @property
    def varIndexByCol(self) -> np.ndarray:
        return self._download("maps")[1]

    @property
    def rowByVarIndex(self) -> np.ndarray:
        vr, vc = self._download("maps")
        n = max(int(vr.max(initial=-1)), int(vc.max(initial=-1))) + 1
        out = np.full(n, -1, dtype=np.int32)
        for r in range(1, len(vr)):
            out[vr[r]] = r
        return out

    @property
    def colByVarIndex(self) -> np.ndarray:
        vr, vc = self._download("maps")
        n = max(int(vr.max(initial=-1)), int(vc.max(initial=-1))) + 1
        out = np.full(n, -1, dtype=np.int32)
        for c in range(1, len(vc)):
            out[vc[c]] = c
        return out

    def final_state(self):
        """(right-hand-side column, cost row, varIndexByRow, varIndexByCol) in one read-back."""
        H, W = self.height, self.width
        rhs, cost = np.empty(H, dtype=np.float64), np.empty(W, dtype=np.float64)
        vr, vc = np.empty(H, dtype=np.int32), np.empty(W, dtype=np.int32)
        _lib.check(self.context.lib.jslp_download(self._h(), None, rhs.ctypes.data, cost.ctypes.data, vr.ctypes.data,
                                                  vc.ctypes.data, None, None, None))
        return rhs, cost, vr, vc

    def sensitivity_bounds(self):
        """jslp_sensitivity: (col_lo, col_hi) over the columns and (row_lo, row_hi) over the rows of the current
        tableau, the ratio-test bounds the sensitivity report is built from (DESIGN.md section 2b)."""
        H, W = self.height, self.width
        col_lo, col_hi = np.empty(W, dtype=np.float64), np.empty(W, dtype=np.float64)
        row_lo, row_hi = np.empty(H, dtype=np.float64), np.empty(H, dtype=np.float64)
        _lib.check(self.context.lib.jslp_sensitivity(self._h(), col_lo.ctypes.data, col_hi.ctypes.data,
                                                     row_lo.ctypes.data, row_hi.ctypes.data))
        return col_lo, col_hi, row_lo, row_hi

    def feasibility_batch(self, keep):
        """jslp_feasibility_batch: phase 1 (cycle check on) of the row subsets keep[s] (n_sets x height, nonzero =
        keep; row 0 is always kept) of the saved snapshot.  Returns (verdict, pivots) int32 arrays, verdict 0 =
        feasible, 1 = infeasible, 2 = undecided (DESIGN.md section 2c).  Leaves the tableau equal to its snapshot."""
        keep = np.ascontiguousarray(keep, dtype=np.uint8)
        n = keep.shape[0]
        verdict, pivots = np.empty(n, dtype=np.int32), np.empty(n, dtype=np.int32)
        _lib.check(self.context.lib.jslp_feasibility_batch(self._h(), keep.ctypes.data, n, verdict.ctypes.data,
                                                           pivots.ctypes.data))
        self._refresh_dims()
        return verdict, pivots

    def parametric_path(self, kind: int, labels, signs, theta0: float, target: float, max_breaks: int) -> dict:
        """jslp_parametric: the breakpoint records of the path of one right-hand side (kind 0) or one cost (kind 1)
        from theta0 to target (DESIGN.md section 2d), the stop code, and column 0 and the row labels at its end.
        The device tableau is restored before the call returns."""
        H = self.height
        lab = np.ascontiguousarray(labels, dtype=np.int32)
        sg = np.ascontiguousarray(signs, dtype=np.float64)
        theta, obj, dobj = (np.empty(max_breaks, dtype=np.float64) for _ in range(3))
        rc = np.empty((max_breaks, 4), dtype=np.int32)
        end_rhs, end_vrow = np.empty(H, dtype=np.float64), np.empty(H, dtype=np.int32)
        n, stop = C.c_int(), C.c_int()
        _lib.check(self.context.lib.jslp_parametric(
            self._h(), int(kind), lab.ctypes.data, sg.ctypes.data, len(lab), float(theta0), float(target),
            int(max_breaks), theta.ctypes.data, obj.ctypes.data, dobj.ctypes.data, rc.ctypes.data, C.byref(n),
            C.byref(stop), end_rhs.ctypes.data, end_vrow.ctypes.data))
        k = n.value
        return {"theta": theta[:k], "obj_raw": obj[:k], "dobj": dobj[:k], "rc_lbl": rc[:k], "stop": stop.value,
                "end_rhs": end_rhs, "end_vrow": end_vrow}

    def frontier_path(self, cost2_by_label, max_breaks: int, max_points: Optional[int] = None) -> dict:
        """jslp_frontier: the second objective priced against the current optimal tableau (R2 and the direction E), the
        breakpoint records of the weight path from 0 to 1 (DESIGN.md section 2g), the stop code, every point on the
        path (column 0, row labels and the record count before it) and the end state.  The device tableau is restored
        before the call returns."""
        H, W = self.height, self.width
        c2 = np.ascontiguousarray(cost2_by_label, dtype=np.float64)
        if len(c2) != self.nVars:
            raise ValueError(f"frontier: the objective has {len(c2)} entries, the tableau {self.nVars} labels")
        # room for a point per breakpoint: np.empty only reserves address space, and the library writes the points
        # the path has; beyond 1 GiB a longer path runs again with room for all of them
        cap = min(max_breaks + 1, max(1, (1 << 30) // (12 * H))) if max_points is None else int(max_points)
        while True:
            r2, dirn = np.empty(W, dtype=np.float64), np.empty(W, dtype=np.float64)
            theta, obj, dobj = (np.empty(max_breaks, dtype=np.float64) for _ in range(3))
            rc = np.empty((max_breaks, 4), dtype=np.int32)
            pt_rhs, pt_vrow = np.empty((max(1, cap), H), dtype=np.float64), np.empty((max(1, cap), H), dtype=np.int32)
            pt_at = np.empty(max(1, cap), dtype=np.int32)
            end_rhs, end_vrow = np.empty(H, dtype=np.float64), np.empty(H, dtype=np.int32)
            n, stop, npts = C.c_int(), C.c_int(), C.c_int()
            _lib.check(self.context.lib.jslp_frontier(
                self._h(), c2.ctypes.data, int(max_breaks), int(cap), r2.ctypes.data, dirn.ctypes.data,
                theta.ctypes.data, obj.ctypes.data, dobj.ctypes.data, rc.ctypes.data, C.byref(n), C.byref(stop),
                pt_rhs.ctypes.data, pt_vrow.ctypes.data, pt_at.ctypes.data, C.byref(npts), end_rhs.ctypes.data,
                end_vrow.ctypes.data))
            if npts.value <= cap or max_points is not None:
                break
            cap = npts.value  # the path is deterministic: run it again with room for every point
        k, p = n.value, min(npts.value, cap)
        return {"r2": r2, "dir": dirn, "theta": theta[:k], "obj_raw": obj[:k], "dobj": dobj[:k], "rc_lbl": rc[:k],
                "stop": stop.value, "pt_rhs": pt_rhs[:p], "pt_vrow": pt_vrow[:p], "pt_break": pt_at[:p],
                "n_points": npts.value, "end_rhs": end_rhs, "end_vrow": end_vrow}

    def scenario_batch(self, edits, offsets, check_cycles: Optional[bool] = None) -> dict:
        """jslp_scenario_batch: edits = [(kind, index, difference), ...] with kind 0 = updateRightHandSide and 1 =
        updateCost; scenario s = edits[offsets[s]:offsets[s + 1]] applied to the current tableau, then simplex() (the
        model's cycle check unless check_cycles is given), each from the current tableau (DESIGN.md section 2e).
        Returns the per-scenario status (0 optimal, 1 infeasible, 2 unbounded, 3 cycled), raw evaluation, phase-1 /
        phase-2 pivots, and the final right-hand-side column and row labels (n x height).  The tableau is unchanged."""
        n, H = len(offsets) - 1, self.height
        arr = (ScenarioEdit * max(1, len(edits)))()
        for i, (kind, index, difference) in enumerate(edits):
            arr[i].kind, arr[i].index, arr[i].difference = int(kind), int(index), float(difference)
        off = np.ascontiguousarray(offsets, dtype=np.int32)
        status, p1, p2 = (np.empty(n, dtype=np.int32) for _ in range(3))
        eval_raw = np.empty(n, dtype=np.float64)
        rhs, vrow = np.empty((n, H), dtype=np.float64), np.empty((n, H), dtype=np.int32)
        cc = self._check_cycles() if check_cycles is None else int(bool(check_cycles))
        _lib.check(self.context.lib.jslp_scenario_batch(
            self._h(), arr, off.ctypes.data, n, cc, status.ctypes.data, eval_raw.ctypes.data, p1.ctypes.data,
            p2.ctypes.data, rhs.ctypes.data, vrow.ctypes.data))
        return {"status": status, "eval_raw": eval_raw, "p1": p1, "p2": p2, "rhs": rhs, "vrow": vrow}

    def recourse_batch(self, edits, offsets, rows, tech) -> dict:
        """jslp_recourse_batch: scenario_batch's run of edits / offsets (cycle check on) and outputs, plus each
        scenario's certificate: "cert_rhs" (column 0 of row 0 at an optimum, of the row phase 1 stopped at when
        infeasible, NaN otherwise) and "alpha" (n x n_first), the certificate row's multipliers of the row labels `rows`
        summed against `tech` -- one matrix (len(rows) x n_first) for every scenario, or one per scenario (n x len(rows)
        x n_first) -- in the rows' tableau sign (DESIGN.md section 2u).  The tableau is unchanged."""
        n, H = len(offsets) - 1, self.height
        arr = self._edit_array([(edits, ())])
        off = np.ascontiguousarray(offsets, dtype=np.int32)
        lab = np.ascontiguousarray(rows, dtype=np.int32)
        tec = np.ascontiguousarray(tech, dtype=np.float64)
        per_case = int(tec.ndim == 3)
        n_first = tec.shape[-1]
        status, p1, p2 = (np.empty(n, dtype=np.int32) for _ in range(3))
        eval_raw, cert_rhs = np.empty(n, dtype=np.float64), np.empty(n, dtype=np.float64)
        rhs, vrow = np.empty((n, H), dtype=np.float64), np.empty((n, H), dtype=np.int32)
        alpha = np.empty((n, n_first), dtype=np.float64)
        _lib.check(self.context.lib.jslp_recourse_batch(
            self._h(), arr, off.ctypes.data, n, lab.ctypes.data if len(lab) else None, len(lab),
            tec.ctypes.data if tec.size else None, n_first, per_case, status.ctypes.data, eval_raw.ctypes.data,
            p1.ctypes.data, p2.ctypes.data, rhs.ctypes.data, vrow.ctypes.data, cert_rhs.ctypes.data,
            alpha.ctypes.data if alpha.size else None))
        return {"status": status, "eval_raw": eval_raw, "p1": p1, "p2": p2, "rhs": rhs, "vrow": vrow,
                "cert_rhs": cert_rhs, "alpha": alpha}

    def _adopt(self, h) -> "GpuTableau":
        """A GpuTableau over the tab handle h that the library derived from this one (face, bound, lex_next, elastic,
        cone): this tableau's precision, context, model, integer count, engine and options, no optional objectives,
        and its size and labels as the library set them."""
        c = GpuTableau(self.precision, context=self.context)
        c.handle = h
        c.model, c.variablesPerIndex = self.model, self.variablesPerIndex
        c.nOpt, c.nInts = 0, getattr(self, "nInts", 0)
        c.engine, c.options = self.engine, dict(self.options)
        c._refresh_dims()
        return c

    def face(self):
        """jslp_face_create: (face, kept columns).  `face` is a GpuTableau of the optimal face of the current (optimal)
        tableau -- the columns whose cost entry lies within the precision, under a zero cost row, with this
        tableau's row labels, options and model (DESIGN.md section 2h) -- or None when only column 0 is kept.  The
        copy stays on the device; this tableau is only read.  close() the face when done."""
        L = self.context.lib
        h, n = C.c_void_p(), C.c_int32()
        kept = np.empty(self.width, dtype=np.int32)
        _lib.check(L.jslp_face_create(self._h(), C.byref(h), C.byref(n), kept.ctypes.data))
        kept = kept[:n.value].copy()
        if not h.value:
            return None, kept
        return self._adopt(h), kept

    def bound(self, allowance: float) -> "GpuTableau":
        """jslp_bound_create: a GpuTableau of the current (optimal) tableau with its objective turned into one bound
        row -- the rows below the cost row unchanged, a zero cost row, and a last row whose slack is `allowance` minus
        the objective a point gives up against the optimum -- with this tableau's column labels, options and model
        and one new row label, max(nVars, lastElementIndex) (DESIGN.md section 2i).  The copy stays on the device;
        this tableau is only read.  close() the bound tableau when done."""
        L = self.context.lib
        h = C.c_void_p()
        _lib.check(L.jslp_bound_create(self._h(), float(allowance), C.byref(h)))
        return self._adopt(h)

    def lex_next(self, cost_by_label, allowance: float):
        """jslp_lex_next: (next, kept columns).  `next` is the starting tableau of the next level of a lexicographic
        chain (DESIGN.md section 2j): face() for allowance == 0, bound(allowance) for allowance > 0, with row 0 the
        objective `cost_by_label` (one entry per label, nVars) priced against the current basis; None when a face
        keeps only column 0.  The copy and row 0 stay on the device; this tableau is only read.  close() it when
        done."""
        c = np.ascontiguousarray(cost_by_label, dtype=np.float64)
        if len(c) != self.nVars:
            raise ValueError(f"lex_next: the objective has {len(c)} entries, the tableau {self.nVars} labels")
        L = self.context.lib
        h, n = C.c_void_p(), C.c_int32()
        kept = np.empty(self.width, dtype=np.int32)
        _lib.check(L.jslp_lex_next(self._h(), c.ctypes.data, float(allowance), C.byref(h), C.byref(n),
                                   kept.ctypes.data))
        kept = kept[:n.value].copy()
        if not h.value:
            return None, kept
        return self._adopt(h), kept

    def elastic(self, rows, weights):
        """jslp_elastic_create: (elastic, crashed).  `elastic` is a GpuTableau of this tableau, as upload() left it,
        with one violation column per row of `rows` (increasing, in 1..height-1) weighted by `weights`, the rows that
        start infeasible crashed onto their column, and row 0 the weighted total violation (DESIGN.md section 2k).  Its
        labels are this tableau's plus len(rows) new ones from max(nVars, lastElementIndex); `crashed` counts the
        crashed rows.  The copy stays on the device; this tableau is only read.  close() it when done."""
        r = np.ascontiguousarray(rows, dtype=np.int32)
        w = np.ascontiguousarray(weights, dtype=np.float64)
        if len(r) != len(w):
            raise ValueError(f"elastic: {len(r)} rows but {len(w)} weights")
        h, n = C.c_void_p(), C.c_int32()
        _lib.check(self.context.lib.jslp_elastic_create(self._h(), r.ctypes.data if len(r) else None,
                                                        w.ctypes.data if len(w) else None, len(r), C.byref(h),
                                                        C.byref(n)))
        return self._adopt(h), n.value

    def cone(self) -> "GpuTableau":
        """jslp_cone_create: a GpuTableau of the recession cone of this tableau, as upload() left it -- column 0 set to
        +0, and one last row sum_j d_j <= 1 over the columns with one new row label, max(nVars, lastElementIndex) --
        with this tableau's column labels, options and model (DESIGN.md section 2l).  The copy stays on the device;
        this tableau is only read.  close() it when done."""
        h = C.c_void_p()
        _lib.check(self.context.lib.jslp_cone_create(self._h(), C.byref(h)))
        return self._adopt(h)

    def column_batch(self, keep_cols) -> dict:
        """jslp_column_batch: simplex() (cycle check on) of the saved snapshot with the columns not kept in keep[s]
        (n_sets x width, nonzero = keep; column 0 is always kept) set to +0 in every row (DESIGN.md section 2l).
        Returns the per-set status (0 optimal, 1 unbounded, 2 cycled, 3 infeasible), raw M[0,0], pivots, and the final
        right-hand-side column and row labels (n x height).  Leaves the tableau equal to its snapshot."""
        keep = np.ascontiguousarray(keep_cols, dtype=np.uint8)
        n, H = keep.shape[0], self.height
        if n and keep.shape[1] != self.width:
            raise ValueError(f"column_batch: masks have {keep.shape[1]} columns, the tableau {self.width}")
        status, pivots = np.empty(n, dtype=np.int32), np.empty(n, dtype=np.int32)
        eval_raw = np.empty(n, dtype=np.float64)
        rhs, vrow = np.empty((n, H), dtype=np.float64), np.empty((n, H), dtype=np.int32)
        _lib.check(self.context.lib.jslp_column_batch(self._h(), keep.ctypes.data, n, status.ctypes.data,
                                                      eval_raw.ctypes.data, pivots.ctypes.data, rhs.ctypes.data,
                                                      vrow.ctypes.data))
        self._refresh_dims()
        return {"status": status, "eval_raw": eval_raw, "pivots": pivots, "rhs": rhs, "vrow": vrow}

    def pool_batch(self, regions, check_cycles: Optional[bool] = None) -> dict:
        """jslp_pool_batch: the region LPs of a solution-pool search (DESIGN.md section 2m).  regions = [(fixings,
        cuts), ...] with fixings [(column, value), ...] applied in order to the saved snapshot and cuts [(type, varIndex,
        value), ...] appended as addCutConstraints appends them, then simplex() (the model's cycle check unless
        check_cycles is given).  Returns the per-region status (0 optimal, 1 infeasible, 2 unbounded, 3 cycled),
        evaluation, is_integral, branch_var / branch_value, pivots, and rhs / vrow (n x row_stride, written for
        integral regions: the final column 0 and row labels, height + len(cuts) entries).  Leaves the tableau equal to
        its snapshot."""
        fixes = (_lib.Fix * max(1, sum(len(fx) for fx, _ in regions)))()
        k = 0
        for fx, _ in regions:
            for col, value in fx:
                fixes[k].column, fixes[k].value = int(col), float(value)
                k += 1
        return self._node_batch(self.context.lib.jslp_pool_batch, fixes, regions, check_cycles)

    def target_batch(self, nodes, check_cycles: Optional[bool] = None) -> dict:
        """jslp_target_batch: the node LPs of the bounding searches of a MIP's near-optimal variability (DESIGN.md
        section 2o).  nodes = [(edits, cuts), ...] with edits [(1, label, difference), ...] applied in order to the
        saved snapshot as updateCost applies them, then the cuts appended and simplex() run as pool_batch does.
        Returns what pool_batch returns.  Leaves the tableau equal to its snapshot."""
        return self._node_batch(self.context.lib.jslp_target_batch, self._edit_array(nodes), nodes, check_cycles)

    def box_batch(self, nodes, check_cycles: Optional[bool] = None) -> dict:
        """jslp_box_batch: the node LPs of the box searches of a two-objective MIP's frontier (DESIGN.md section 2s).
        nodes = [(edits, cuts), ...] with edits [(kind, label, difference), ...] -- kind 0 = updateRightHandSide, before
        any kind 1 = updateCost -- applied in order to the saved snapshot, then the cuts appended and simplex() run as
        pool_batch does.  Returns what pool_batch returns.  Leaves the tableau equal to its snapshot."""
        return self._node_batch(self.context.lib.jslp_box_batch, self._edit_array(nodes), nodes, check_cycles)

    @staticmethod
    def _edit_array(nodes):
        """The edits of nodes = [(edits of node i, cuts of node i), ...] as one ctypes array, in node order."""
        arr = (ScenarioEdit * max(1, sum(len(ed) for ed, _ in nodes)))()
        k = 0
        for ed, _ in nodes:
            for kind, index, difference in ed:
                arr[k].kind, arr[k].index, arr[k].difference = int(kind), int(index), float(difference)
                k += 1
        return arr

    def _node_batch(self, fn, edits, nodes, check_cycles: Optional[bool]) -> dict:
        """The call and outputs jslp_pool_batch, jslp_target_batch and jslp_box_batch share: edits (a ctypes array) in
        the order of nodes = [(edits of node i, cuts of node i), ...]."""
        n = len(nodes)
        edit_off, cut_off = np.zeros(n + 1, dtype=np.int32), np.zeros(n + 1, dtype=np.int32)
        for i, (ed, cs) in enumerate(nodes):
            edit_off[i + 1], cut_off[i + 1] = edit_off[i] + len(ed), cut_off[i] + len(cs)
        cuts = self._cut_array([c for _, cs in nodes for c in cs])
        stride = self.height + max((len(cs) for _, cs in nodes), default=0)
        status, integral, bvar, pivots = (np.empty(n, dtype=np.int32) for _ in range(4))
        evaluation, bval = np.empty(n, dtype=np.float64), np.empty(n, dtype=np.float64)
        rhs, vrow = np.zeros((n, stride), dtype=np.float64), np.zeros((n, stride), dtype=np.int32)
        cc = self._check_cycles() if check_cycles is None else int(bool(check_cycles))
        _lib.check(fn(self._h(), edits, edit_off.ctypes.data, cuts, cut_off.ctypes.data, n, cc, stride,
                      status.ctypes.data, evaluation.ctypes.data, integral.ctypes.data, bvar.ctypes.data,
                      bval.ctypes.data, pivots.ctypes.data, rhs.ctypes.data, vrow.ctypes.data))
        self._refresh_dims()
        return {"status": status, "evaluation": evaluation, "is_integral": integral, "branch_var": bvar,
                "branch_value": bval, "pivots": pivots, "rhs": rhs, "vrow": vrow}

    def conflict_batch(self, keep, int_keep, cuts) -> dict:
        """jslp_conflict_batch: the node LPs of a MIP conflict search (DESIGN.md section 2n).  keep (n x height,
        nonzero = keep; row 0 is always kept) selects rows of the saved snapshot, int_keep (n x integer variables, in
        integerIndices order) the integrality the scan checks, and cuts[i] = [(type, varIndex, value), ...] the cut
        rows appended after the kept rows; then phase 1 with the cycle check on.  Returns the per-node status (0
        feasible, 1 infeasible, 2 cycled), is_integral, branch_var / branch_value, pivots, and rhs / vrow (n x
        row_stride: the final column 0 and row labels, 1 + kept rows + cuts entries, unless the node cycled).  Leaves
        the tableau equal to its snapshot."""
        keep = np.ascontiguousarray(keep, dtype=np.uint8)
        int_keep = np.ascontiguousarray(int_keep, dtype=np.uint8)
        n = keep.shape[0]
        cut_off = np.zeros(n + 1, dtype=np.int32)
        for i, cs in enumerate(cuts):
            cut_off[i + 1] = cut_off[i] + len(cs)
        arr = self._cut_array([c for cs in cuts for c in cs])
        stride = int(keep[:, 1:].astype(bool).sum(axis=1).max(initial=0)) + 1 + max((len(cs) for cs in cuts), default=0)
        status, integral, bvar, pivots = (np.empty(n, dtype=np.int32) for _ in range(4))
        bval = np.empty(n, dtype=np.float64)
        rhs, vrow = np.zeros((n, stride), dtype=np.float64), np.zeros((n, stride), dtype=np.int32)
        _lib.check(self.context.lib.jslp_conflict_batch(
            self._h(), keep.ctypes.data, int_keep.ctypes.data if int_keep.size else None, arr, cut_off.ctypes.data, n,
            stride, status.ctypes.data, integral.ctypes.data, bvar.ctypes.data, bval.ctypes.data, pivots.ctypes.data,
            rhs.ctypes.data, vrow.ctypes.data))
        self._refresh_dims()
        return {"status": status, "is_integral": integral, "branch_var": bvar, "branch_value": bval,
                "pivots": pivots, "rhs": rhs, "vrow": vrow}

    def column(self, col: int) -> np.ndarray:
        """jslp_column: column `col` of the current tableau (height doubles), without downloading the rest."""
        out = np.empty(self.height, dtype=np.float64)
        _lib.check(self.context.lib.jslp_column(self._h(), int(col), out.ctypes.data))
        return out

    def crash(self, enter, leave):
        """jslp_crash: pivot the labels `enter` into the basis in order, each on the row with the largest |entry| among
        the rows whose basic label has leave[label] != 0 (DESIGN.md section 2f).  Returns the records (n x 4: label,
        row, column, leaving label or -1 rejected / -2 already basic) and the number of pivots done."""
        ent = np.ascontiguousarray(enter, dtype=np.int32)
        lv = np.ascontiguousarray(leave, dtype=np.uint8)
        if len(lv) != self.nVars:
            raise ValueError(f"crash: the leave mask has {len(lv)} entries, the tableau {self.nVars} labels")
        out = np.empty((max(1, len(ent)), 4), dtype=np.int32)
        n = C.c_int()
        _lib.check(self.context.lib.jslp_crash(self._h(), ent.ctypes.data if len(ent) else None, len(ent),
                                               lv.ctypes.data if len(lv) else None, out.ctypes.data, C.byref(n)))
        self._edited()
        return out[:len(ent)], n.value

    def optional_reduced_costs(self) -> np.ndarray:
        return self._download("opt")

    def pivot_log(self) -> np.ndarray:
        """All pivots executed on this tableau since upload (row, col, leaving var, entering var);
        needs JSLP_OPT_PIVOT_LOG_CAP.  The library hands the log over in drains; they are
        accumulated here."""
        n = C.c_int()
        L = self.context.lib
        cap = 1 << 20
        buf = np.empty((cap, 4), dtype=np.int32)
        _lib.check(L.jslp_pivot_log(self._h(), buf.ctypes.data, cap, C.byref(n)))
        new = buf[:min(cap, n.value)].copy()
        old = self._cache_log if self._cache_log is not None else np.empty((0, 4), dtype=np.int32)
        self._cache_log = np.concatenate([old, new]) if len(new) else old
        return self._cache_log

    # ------------------------------------------------------------------ solve (tableau.ts:250-274)
    def updateVariableValues(self) -> None:  # dynamic-modification.ts:57-76
        if self.model is None or self.handle is None:
            return
        rhs = self.rhs_column()
        row_of = self.rowByVarIndex
        rounding = js_round(1 / self.precision)
        for var in self.model.variables:
            r = row_of[var.index] if var.index < len(row_of) else -1
            var.value = 0 if r == -1 else js_round((float(rhs[r]) + EPSILON) * rounding) / rounding

    def solve(self, start=None, start_nodes: int = 1000):
        if self.model is not None and self.model.getNumberOfIntegerVariables() > 0:
            self.branchAndCut(start, start_nodes)
        else:
            self.simplex()
        self.updateVariableValues()
        return self.getSolution()

    def getSolution(self):
        is_min = True if self.model is None else self.model.isMinimization
        evaluation = self.evaluation if is_min else -self.evaluation
        if self.model is not None and self.model.getNumberOfIntegerVariables() > 0:
            return MilpSolution(self, evaluation, self.feasible, self.bounded, self.branchAndCutIterations)
        return Solution(self, evaluation, self.feasible, self.bounded)

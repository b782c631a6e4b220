"""oracle/ref_model.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement of the reference's JSON front end and result shaping, driving the C
restatement of the numeric core (oracle/jslp_oracle.c) through ctypes.  Together they are
the checker for the CUDA path.  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this module.

Reference code restated (all under /root/reference/src/):
  model.ts:278-419      Model.loadJson (row/column ordering, binaries -> rows, options)
  model.ts:427-467      Model.solve + applyPresolveReductions
  expressions.ts:73-94,96-203,205-247  relaxation variables, Constraint, Equality
  tableau/presolve.ts:179-306,320-492  presolve passes
  tableau/tableau.ts:278-391           setOptionalObjective, initialize, _resetMatrix, setModel
  tableau/tableau.ts:250-274           solve / getSolution
  tableau/dynamic-modification.ts:57-76 updateVariableValues
  tableau/solution.ts:35-60            generateSolutionSet
  main.ts:94-147,173-193               Solve / buildSimplifiedResult

JS semantics that matter and are restated explicitly: Object.keys order (canonical array
indices first, ascending), Math.round (ties toward +inf), Number.EPSILON, truthiness (`||`).
"""
from __future__ import annotations

import ctypes
import math
import os
import subprocess
from typing import Any

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

EPSILON = 2.220446049250313e-16


def build_oracle(force: bool = False) -> str:
    so = os.path.join(_HERE, "libjslp_oracle.so")
    src = os.path.join(_HERE, "jslp_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-B", "libjslp_oracle.so"])
    return so


class OrcCut(ctypes.Structure):
    _fields_ = [("type", ctypes.c_int), ("varIndex", ctypes.c_int), ("value", ctypes.c_double)]


class OrcState(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in (
        "width", "height", "nVars", "lastElementIndex", "feasible", "bounded", "simplexIters",
        "unboundedVar", "isIntegral", "bncIterations", "cyclePhase", "cycleStart", "cycleLen",
        "nBestCuts")] + [(n, ctypes.c_int64) for n in (
        "totalPivots", "lastP1", "lastP2", "plogN", "nlogN")] + [
        ("evaluation", ctypes.c_double), ("bestPossibleEval", ctypes.c_double)]


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build_oracle())
        L.orc_create.restype = ctypes.c_void_p
        L.orc_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_double]
        for name in ("orc_destroy", "orc_simplex", "orc_save", "orc_restore", "orc_branch_and_cut"):
            getattr(L, name).argtypes = [ctypes.c_void_p]
            getattr(L, name).restype = None
        for name in ("orc_phase1", "orc_phase2"):
            getattr(L, name).argtypes = [ctypes.c_void_p]
            getattr(L, name).restype = ctypes.c_long
        L.orc_upload.argtypes = [ctypes.c_void_p] + [ctypes.c_void_p] * 3
        L.orc_set_unrestricted.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.orc_set_integers.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.orc_set_optional.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        L.orc_set_options.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                      ctypes.c_double, ctypes.c_long]
        L.orc_enable_pivot_log.argtypes = [ctypes.c_void_p, ctypes.c_long]
        L.orc_enable_node_log.argtypes = [ctypes.c_void_p, ctypes.c_long]
        L.orc_pivot.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        L.orc_add_cuts.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.orc_apply_cuts.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.orc_is_integral.argtypes = [ctypes.c_void_p]
        L.orc_is_integral.restype = ctypes.c_int
        L.orc_most_fractional.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_double)]
        L.orc_most_fractional.restype = ctypes.c_int
        L.orc_get_state.argtypes = [ctypes.c_void_p, ctypes.POINTER(OrcState)]
        for name in ("orc_get_matrix", "orc_get_optional", "orc_get_pivot_log", "orc_get_node_log",
                     "orc_get_best_cuts"):
            getattr(L, name).argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.orc_get_maps.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.orc_get_flat.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long]
        L.orc_row_of.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.orc_row_of.restype = ctypes.c_int
        L.orc_set_flags.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        L.orc_set_pivot_limit.argtypes = [ctypes.c_void_p, ctypes.c_long]
        L.orc_set_use_mir.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.orc_enhanced_branch_and_cut.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.orc_enhanced_branch_and_cut.restype = None
        L.orc_enhanced_branch_and_cut2.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 5
        L.orc_enhanced_branch_and_cut2.restype = None
        for name in ("orc_dm_put_in_base", "orc_dm_take_out_of_base", "orc_dm_remove_constraint", "orc_dm_remove_variable"):
            getattr(L, name).argtypes = [ctypes.c_void_p, ctypes.c_int]
            getattr(L, name).restype = ctypes.c_int
        L.orc_dm_update_rhs.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_double]
        L.orc_dm_update_coefficient.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double]
        L.orc_dm_update_coefficient.restype = ctypes.c_int
        L.orc_dm_update_cost.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double]
        L.orc_dm_add_constraint.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_int]
        L.orc_dm_add_variable.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_int]
        L.orc_add_mir_cut.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        L.orc_add_mir_cut.restype = ctypes.c_int
        L.orc_apply_mir_cuts.argtypes = [ctypes.c_void_p]
        L.orc_apply_mir_cuts.restype = ctypes.c_int
        L.orc_fractional_volume.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.orc_fractional_volume.restype = ctypes.c_double
        L.orc_truncated.argtypes = [ctypes.c_void_p]
        L.orc_truncated.restype = ctypes.c_int
        L.orc_cycles_ref.argtypes = [ctypes.c_void_p, ctypes.c_long,
                                     ctypes.POINTER(ctypes.c_long), ctypes.POINTER(ctypes.c_long)]
        L.orc_cycles_fast.argtypes = L.orc_cycles_ref.argtypes
        _LIB = L
    return _LIB


# ---------------------------------------------------------------- JS semantics helpers
def js_keys(d: dict) -> list[str]:
    """Object.keys order: canonical array-index keys ascending, then insertion order."""
    idx, rest = [], []
    for k in d.keys():
        if k.isdigit() and (k == "0" or k[0] != "0") and int(k) < 4294967295:
            idx.append(k)
        else:
            rest.append(k)
    idx.sort(key=int)
    return idx + rest


def js_round(x: float) -> float:
    if x != x or math.isinf(x):
        return x
    f = math.floor(x)
    return float(f + 1) if x - f >= 0.5 else float(f)


def js_div(a: float, b: float) -> float:
    """IEEE division as JS does it (no ZeroDivisionError)."""
    if b == 0:
        if a == 0 or a != a:
            return math.nan
        return math.copysign(math.inf, a) * math.copysign(1.0, b)
    return a / b


def js_truthy(v: Any) -> bool:
    if v is None or v is False:
        return False
    if isinstance(v, (int, float)) and not isinstance(v, bool):
        return not (v == 0 or v != v)
    if isinstance(v, str):
        return v != ""
    return True


# ---------------------------------------------------------------- expressions.ts
class Variable:
    def __init__(self, vid, cost, index, priority, is_integer=False, is_slack=False):
        self.id, self.cost, self.index, self.priority = vid, cost, index, priority
        self.value = 0.0
        self.isInteger = is_integer
        self.isSlack = is_slack


class Term:
    def __init__(self, variable, coefficient):
        self.variable, self.coefficient = variable, coefficient


class Constraint:
    def __init__(self, rhs, is_upper, index, model):
        self.slack = Variable("s" + str(index), 0, index, 0, is_slack=True)
        self.index, self.model, self.rhs, self.isUpperBound = index, model, rhs, is_upper
        self.terms: list[Term] = []
        self.termsByVarIndex: dict[int, Term] = {}
        self.relaxation = None

    def addTerm(self, coefficient, variable):  # expressions.ts:119-137
        term = self.termsByVarIndex.get(variable.index)
        if term is None:
            t = Term(variable, coefficient)
            self.termsByVarIndex[variable.index] = t
            self.terms.append(t)
        else:
            self.setVariableCoefficient(term.coefficient + coefficient, variable)
        return self

    def setVariableCoefficient(self, new_coefficient, variable):  # expressions.ts:158-184
        term = self.termsByVarIndex.get(variable.index)
        if term is None:
            self.addTerm(new_coefficient, variable)
        elif new_coefficient != term.coefficient:
            term.coefficient = new_coefficient
        return self

    def relax(self, weight, priority):  # expressions.ts:186-202
        self.relaxation = create_relaxation_variable(self.model, weight, priority)
        self._relax(self.relaxation)

    def _relax(self, rv):
        if rv is None:
            return
        self.setVariableCoefficient(-1 if self.isUpperBound else 1, rv)


def create_relaxation_variable(model, weight, priority):  # expressions.ts:73-94
    if priority == 0 or priority == "required":
        return None
    w = 1 if weight is None else weight
    p = 1 if priority is None else priority
    actual = -w if model.isMinimization is False else w
    rid = "r" + str(model.relaxationIndex)
    model.relaxationIndex += 1
    return model.addVariable(actual, rid, False, False, p)


# ---------------------------------------------------------------- model.ts
class RefModel:
    def __init__(self, precision=None):
        self.precision = 1e-8 if precision is None else precision  # tableau.ts:96
        self.variables: list[Variable] = []
        self.integerVariables: list[Variable] = []
        self.unrestrictedVariables: dict[int, bool] = {}
        self.constraints: list[Constraint] = []
        self.isMinimization = True
        self.relaxationIndex = 1
        self.useMIRCuts = False
        self.checkForCycles = True
        self.tolerance = 0
        self.timeout = None
        self.keep_solutions = False
        self.usePresolve = True
        self.lastElementIndex = 0  # Tableau.getNewElementIndex counter before initialize
        self.variablesPerIndex: dict[int, Variable] = {}
        self.presolve_infeasible = False
        self.fixed: dict[Variable, float] = {}

    def _new_index(self):
        i = self.lastElementIndex
        self.lastElementIndex += 1
        return i

    def _add_constraint(self, rhs, is_upper):
        c = Constraint(rhs, is_upper, self._new_index(), self)
        self.variablesPerIndex[c.slack.index] = c.slack
        self.constraints.append(c)
        return c

    def smallerThan(self, rhs):
        return self._add_constraint(rhs, True)

    def greaterThan(self, rhs):
        return self._add_constraint(rhs, False)

    def addVariable(self, cost, vid, is_integer, is_unrestricted, priority=None):  # model.ts:136-196
        if isinstance(priority, str):
            priority = {"required": 0, "strong": 1, "medium": 2, "weak": 3}.get(priority, 0)
        idx = self._new_index()
        ident = vid if vid is not None else "v" + str(idx)
        v = Variable(ident, 0 if cost is None else cost, idx, 0 if priority is None else priority,
                     is_integer=bool(is_integer))
        if is_integer:
            self.integerVariables.append(v)
        self.variables.append(v)
        self.variablesPerIndex[idx] = v
        if is_unrestricted:
            self.unrestrictedVariables[idx] = True
        return v

    def loadJson(self, jm: dict):  # model.ts:278-419
        self.isMinimization = jm.get("opType") != "max"
        variables = jm["variables"]
        constraints = jm["constraints"]
        cmin: dict[str, Constraint] = {}
        cmax: dict[str, Constraint] = {}
        for cid in js_keys(constraints):
            cdef = constraints[cid]
            if not isinstance(cdef, dict):
                cdef = {}
            equal = cdef.get("equal")
            weight = cdef.get("weight")
            priority = cdef.get("priority")
            relaxed = weight is not None or priority is not None
            if equal is None:
                mn = cdef.get("min")
                if mn is not None:
                    lb = self.greaterThan(mn)
                    cmin[cid] = lb
                    if relaxed:
                        lb.relax(weight, priority)
                mx = cdef.get("max")
                if mx is not None:
                    ub = self.smallerThan(mx)
                    cmax[cid] = ub
                    if relaxed:
                        ub.relax(weight, priority)
            else:
                lb = self.greaterThan(equal)
                cmin[cid] = lb
                ub = self.smallerThan(equal)
                cmax[cid] = ub
                if relaxed:  # Equality.relax, expressions.ts:240-246
                    rv = create_relaxation_variable(self, weight, priority)
                    lb.relaxation = rv
                    lb._relax(rv)
                    ub.relaxation = rv
                    ub._relax(rv)

        self.tolerance = jm.get("tolerance") if js_truthy(jm.get("tolerance")) else 0
        if js_truthy(jm.get("timeout")):
            self.timeout = jm["timeout"]
        opts = jm.get("options")
        if js_truthy(opts):
            if js_truthy(opts.get("timeout")):
                self.timeout = opts["timeout"]
            if self.tolerance == 0:
                self.tolerance = opts.get("tolerance") if js_truthy(opts.get("tolerance")) else 0
            if js_truthy(opts.get("useMIRCuts")):
                self.useMIRCuts = opts["useMIRCuts"]
            self.checkForCycles = True if "exitOnCycles" not in opts else opts["exitOnCycles"]
            self.keep_solutions = opts["keep_solutions"] if js_truthy(opts.get("keep_solutions")) else False
            if opts.get("presolve") is not None:
                self.usePresolve = opts["presolve"]

        ints = jm.get("ints") or {}
        bins = jm.get("binaries") or {}
        unres = jm.get("unrestricted") or {}
        objective = jm.get("optimize")
        for vid in js_keys(variables):
            vc = variables[vid]
            cost = vc.get(objective) if isinstance(objective, str) else None
            cost = cost if js_truthy(cost) else 0
            is_binary = js_truthy(bins.get(vid))
            is_integer = js_truthy(ints.get(vid)) or is_binary
            is_unres = js_truthy(unres.get(vid))
            var = self.addVariable(cost, vid, is_integer, is_unres)
            if is_binary:
                self.smallerThan(1).addTerm(1, var)
            for cname in js_keys(vc):
                if cname == objective:
                    continue
                coef = vc[cname]
                c = cmin.get(cname)
                if c is not None:
                    c.addTerm(coef, var)
                c = cmax.get(cname)
                if c is not None:
                    c.addTerm(coef, var)
        return self

    # ------------------------------------------------------------ tableau.ts:292-391
    def build_tableau(self):
        """Tableau.setModel: returns (matrix HxW, vrow, vcol, optional priorities, optional rc)."""
        W = len(self.variables) + 1
        H = len(self.constraints) + 1
        M = np.zeros((H, W), dtype=np.float64)
        vrow = np.full(H, -1, dtype=np.int32)
        vcol = np.full(W, -1, dtype=np.int32)
        coeff = -1 if self.isMinimization else 1
        opt: dict[int, np.ndarray] = {}
        col_of: dict[int, int] = {}
        for v, var in enumerate(self.variables):
            cost = coeff * float(var.cost)   # a double product, as in JS: -1 * 0 is -0
            if var.priority == 0:
                M[0, v + 1] = cost
            else:
                if var.priority not in opt:
                    opt[var.priority] = np.zeros(W, dtype=np.float64)
                opt[var.priority][v + 1] = cost
            col_of[var.index] = v + 1
            vcol[v + 1] = var.index
        r = 1
        for c in self.constraints:
            vrow[r] = c.index
            if c.isUpperBound:
                for t in c.terms:
                    M[r, col_of[t.variable.index]] = t.coefficient
                M[r, 0] = c.rhs
            else:
                for t in c.terms:
                    M[r, col_of[t.variable.index]] = -float(t.coefficient)
                M[r, 0] = -float(c.rhs)
            r += 1
        prios = sorted(opt.keys())
        rc = np.stack([opt[p] for p in prios]) if prios else np.zeros((0, W))
        return M, vrow, vcol, prios, rc


# ---------------------------------------------------------------- presolve.ts
def presolve(model: RefModel):
    """Returns (is_infeasible, fixed: dict[Variable, value]).  presolve.ts:320-492."""
    fixed: dict[Variable, float] = {}
    removed: set[int] = set()
    bounds: dict[Variable, dict] = {}  # insertion-ordered like a JS Map

    def falsy(x):
        return x is None or x == 0 or x != x

    def remove_redundant():  # presolve.ts:246-306
        changed = False
        for ci, con in enumerate(model.constraints):
            if ci in removed:
                continue
            mn = 0.0
            mx = 0.0
            for t in con.terms:
                fv = fixed.get(t.variable)
                if fv is not None:
                    mn += t.coefficient * fv
                    mx += t.coefficient * fv
                    continue
                b = bounds.get(t.variable, {})
                lower = b.get("lower") if b.get("lower") is not None else 0
                upper = b.get("upper") if b.get("upper") is not None else math.inf
                big = 1e10 if upper == math.inf else upper
                if t.coefficient > 0:
                    mn += t.coefficient * lower
                    mx += t.coefficient * big
                else:
                    mn += t.coefficient * big
                    mx += t.coefficient * lower
            if con.isUpperBound:
                if mx <= con.rhs + 1e-6:
                    removed.add(ci)
                    changed = True
                if mn > con.rhs + 1e-6:
                    return None
            else:
                if mn >= con.rhs - 1e-6:
                    removed.add(ci)
                    changed = True
                if mx < con.rhs - 1e-6:
                    return None
        return changed

    def tighten_coefficients():  # presolve.ts:179-240
        changed = False
        for ci, con in enumerate(model.constraints):
            if ci in removed or not con.isUpperBound:
                continue
            min_act = 0.0
            for t in con.terms:
                if t.variable in fixed:
                    min_act += t.coefficient * fixed[t.variable]
                else:
                    b = bounds.get(t.variable, {})
                    lower = b.get("lower") if b.get("lower") is not None else 0
                    if t.coefficient > 0:
                        min_act += t.coefficient * lower
                    else:
                        upper = b.get("upper") if b.get("upper") is not None else math.inf
                        min_act += t.coefficient * upper
            slack = con.rhs - min_act
            if slack < 0:
                continue
            for t in con.terms:
                if t.variable in fixed or not t.variable.isInteger or t.coefficient <= 0:
                    continue
                b = bounds.get(t.variable, {})
                lower = b.get("lower") if b.get("lower") is not None else 0
                upper = b.get("upper") if b.get("upper") is not None else 1
                if lower >= -0.5 and upper <= 1.5:
                    eff = t.coefficient * (upper - lower)
                    if eff > slack + 1e-6:
                        implied = lower + slack / t.coefficient
                        if implied < upper - 1e-6:
                            cur = bounds.get(t.variable, {})
                            if falsy(cur.get("upper")) or implied < cur["upper"]:
                                nb = dict(cur)
                                nb["upper"] = implied
                                bounds[t.variable] = nb
                                changed = True
        return changed

    changed = True
    passes = 0
    while changed and passes < 5:
        changed = False
        passes += 1
        for ci, con in enumerate(model.constraints):  # pass 1: singleton rows
            if ci in removed:
                continue
            active = [t for t in con.terms if t.variable not in fixed]
            if len(active) == 0:
                lhs = 0.0
                for t in con.terms:
                    fv = fixed.get(t.variable)
                    if fv is not None:
                        lhs += t.coefficient * fv
                ok = lhs <= con.rhs + 1e-6 if con.isUpperBound else lhs >= con.rhs - 1e-6
                if not ok:
                    return True, fixed
                removed.add(ci)
                changed = True
            elif len(active) == 1:
                term = active[0]
                var, coeff = term.variable, term.coefficient
                rhs_adj = con.rhs
                for t in con.terms:
                    if t.variable is not var:
                        fv = fixed.get(t.variable)
                        if fv is not None:
                            rhs_adj -= t.coefficient * fv
                bound = js_div(rhs_adj, coeff)
                if con.isUpperBound:
                    cur = bounds.get(var)
                    if coeff > 0:
                        if cur is None or falsy(cur.get("upper")) or bound < cur["upper"]:
                            nb = dict(cur) if cur else {}
                            nb["upper"] = bound
                            bounds[var] = nb
                            changed = True
                    else:
                        if cur is None or falsy(cur.get("lower")) or bound > cur["lower"]:
                            nb = dict(cur) if cur else {}
                            nb["lower"] = bound
                            bounds[var] = nb
                            changed = True
                removed.add(ci)
        for var, b in list(bounds.items()):  # pass 2: fixings from bounds
            if var in fixed:
                continue
            lo, up = b.get("lower"), b.get("upper")
            if lo is not None and up is not None:
                if lo > up + 1e-6:
                    return True, fixed
                if abs(lo - up) < 1e-6:
                    fv = lo
                    if var.isInteger:
                        fv = js_round(fv)
                    fixed[var] = fv
                    changed = True
            if var.isInteger and lo is not None and lo >= 0.5:
                if (up if up is not None else math.inf) <= 1.5:
                    fixed[var] = 1
                    changed = True
            if var.isInteger and up is not None and up <= 0.5:
                if (lo if lo is not None else 0) >= -0.5:
                    fixed[var] = 0
                    changed = True
        rr = remove_redundant()
        if rr is None:
            return True, fixed
        if rr:
            changed = True
        if tighten_coefficients():
            changed = True
    return False, fixed


# ---------------------------------------------------------------- oracle tableau wrapper
class OracleTableau:
    """Owns one orc_tab; mirrors the Tableau seam (simplex/pivot/save/restore/branchAndCut)."""

    def __init__(self, M, vrow, vcol, precision=1e-8, unrestricted=None, integers=None,
                 opt_rc=None, check_cycles=True, fast_cycles=False, is_min=True, tolerance=0.0,
                 max_nodes=0, pivot_log=0, node_log=0, use_mir=False):
        L = lib()
        M = np.ascontiguousarray(M, dtype=np.float64)
        self.H0, self.W = M.shape
        self.h = L.orc_create(self.W, self.H0, precision)
        vrow = np.ascontiguousarray(vrow, dtype=np.int32)
        vcol = np.ascontiguousarray(vcol, dtype=np.int32)
        L.orc_upload(self.h, M.ctypes.data, vrow.ctypes.data, vcol.ctypes.data)
        if unrestricted is not None and len(unrestricted):
            u = np.ascontiguousarray(unrestricted, dtype=np.uint8)
            L.orc_set_unrestricted(self.h, u.ctypes.data, len(u))
        if integers is not None and len(integers):
            iv = np.ascontiguousarray(integers, dtype=np.int32)
            L.orc_set_integers(self.h, iv.ctypes.data, len(iv))
        if opt_rc is not None and len(opt_rc):
            rc = np.ascontiguousarray(opt_rc, dtype=np.float64)
            L.orc_set_optional(self.h, rc.shape[0], rc.ctypes.data)
        self.nOpt = 0 if opt_rc is None else len(opt_rc)
        L.orc_set_options(self.h, int(bool(check_cycles)), int(bool(fast_cycles)), int(bool(is_min)),
                          float(tolerance), int(max_nodes))
        L.orc_set_use_mir(self.h, int(bool(use_mir)))
        if pivot_log:
            L.orc_enable_pivot_log(self.h, pivot_log)
        if node_log:
            L.orc_enable_node_log(self.h, node_log)

    def __del__(self):
        if getattr(self, "h", None):
            try:
                lib().orc_destroy(self.h)
            except Exception:  # interpreter shutdown: module globals may already be gone
                pass
            self.h = None

    def set_pivot_limit(self, n):
        lib().orc_set_pivot_limit(self.h, int(n))

    def truncated(self):
        return bool(lib().orc_truncated(self.h))

    def simplex(self):
        lib().orc_simplex(self.h)
        return self.state()

    def phase1(self):
        return lib().orc_phase1(self.h)

    def phase2(self):
        return lib().orc_phase2(self.h)

    def pivot(self, r, c):
        lib().orc_pivot(self.h, r, c)

    def save(self):
        lib().orc_save(self.h)

    def restore(self):
        lib().orc_restore(self.h)

    @staticmethod
    def _cuts(cuts):
        arr = (OrcCut * max(1, len(cuts)))()
        for i, (t, v, val) in enumerate(cuts):
            arr[i].type = 0 if t in (0, "min") else 1
            arr[i].varIndex = v
            arr[i].value = val
        return arr

    def add_cuts(self, cuts):
        lib().orc_add_cuts(self.h, self._cuts(cuts), len(cuts))

    def apply_cuts(self, cuts):
        lib().orc_apply_cuts(self.h, self._cuts(cuts), len(cuts))
        return self.state()

    def branch_and_cut(self):
        lib().orc_branch_and_cut(self.h)
        return self.state()

    NODE_SELECTION = {"best-first": 1, "depth-first": 2, "hybrid": 3}
    BRANCHING = {"most-fractional": 1, "pseudocost": 2, "strong": 3}

    def enhanced_branch_and_cut(self, node_selection="hybrid", branching="pseudocost", strong_candidates=5):
        lib().orc_enhanced_branch_and_cut(self.h, self.NODE_SELECTION[node_selection], self.BRANCHING[branching], strong_candidates)
        return self.state()

    def incremental_branch_and_cut(self, node_selection="hybrid", branching="pseudocost", max_checkpoints=50):
        lib().orc_enhanced_branch_and_cut2(self.h, self.NODE_SELECTION[node_selection], self.BRANCHING[branching], 5, 1, max_checkpoints)
        return self.state()

    # ---- dynamic-modification.ts (indices instead of Constraint / Variable objects)
    def put_in_base(self, var_index):
        return lib().orc_dm_put_in_base(self.h, int(var_index))

    def take_out_of_base(self, var_index):
        return lib().orc_dm_take_out_of_base(self.h, int(var_index))

    def update_rhs(self, constraint_index, difference):
        lib().orc_dm_update_rhs(self.h, int(constraint_index), float(difference))

    def update_coefficient(self, constraint_index, var_index, difference):
        rc = lib().orc_dm_update_coefficient(self.h, int(constraint_index), int(var_index), float(difference))
        if rc == -1:
            raise ValueError("[Tableau.updateConstraintCoefficient] constraint index should not be equal to variable index !")
        return rc

    def update_cost(self, var_index, difference, opt_slot=-1):
        lib().orc_dm_update_cost(self.h, int(var_index), int(opt_slot), float(difference))

    def add_constraint(self, is_upper, rhs, slack_index, terms):
        tv = np.ascontiguousarray([v for v, _ in terms], dtype=np.int32)
        tc = np.ascontiguousarray([c for _, c in terms], dtype=np.float64)
        lib().orc_dm_add_constraint(self.h, int(bool(is_upper)), float(rhs), int(slack_index), tv.ctypes.data, tc.ctypes.data, len(terms))

    def remove_constraint(self, slack_index):
        return lib().orc_dm_remove_constraint(self.h, int(slack_index))

    def add_variable(self, var_index, cost_entry, opt_slot=-1):
        lib().orc_dm_add_variable(self.h, int(var_index), float(cost_entry), int(opt_slot))
        self.W += 1

    def remove_variable(self, var_index):
        rc = lib().orc_dm_remove_variable(self.h, int(var_index))
        if rc == 0:
            self.W -= 1
        return rc

    def add_mir_cut(self, row, upper=False):   # addLowerBoundMIRCut / addUpperBoundMIRCut
        return bool(lib().orc_add_mir_cut(self.h, int(row), int(bool(upper))))

    def apply_mir_cuts(self):                  # applyMIRCuts
        return lib().orc_apply_mir_cuts(self.h)

    def fractional_volume(self, ignore_integer_values=False):  # computeFractionalVolume
        return lib().orc_fractional_volume(self.h, int(bool(ignore_integer_values)))

    def is_integral(self):
        return bool(lib().orc_is_integral(self.h))

    def most_fractional(self):
        v = ctypes.c_double()
        i = lib().orc_most_fractional(self.h, ctypes.byref(v))
        return i, v.value

    def state(self) -> OrcState:
        s = OrcState()
        lib().orc_get_state(self.h, ctypes.byref(s))
        return s

    def matrix(self):
        s = self.state()
        out = np.empty((s.height, s.width), dtype=np.float64)
        lib().orc_get_matrix(self.h, out.ctypes.data)
        return out

    def flat(self, n):
        """The first n doubles of the backing Float64Array, whatever the current width says (removeVariable)."""
        out = np.empty(n, dtype=np.float64)
        lib().orc_get_flat(self.h, out.ctypes.data, n)
        return out

    def maps(self):
        s = self.state()
        vrow = np.empty(s.height, dtype=np.int32)
        vcol = np.empty(s.width, dtype=np.int32)
        lib().orc_get_maps(self.h, vrow.ctypes.data, vcol.ctypes.data)
        return vrow, vcol

    def row_of(self, var_index):
        return lib().orc_row_of(self.h, var_index)

    def optional(self):
        out = np.empty((self.nOpt, self.W), dtype=np.float64)
        lib().orc_get_optional(self.h, out.ctypes.data)
        return out

    def pivot_log(self):
        s = self.state()
        out = np.empty((s.plogN, 4), dtype=np.int32)
        if s.plogN:
            lib().orc_get_pivot_log(self.h, out.ctypes.data)
        return out

    def node_log(self):
        s = self.state()
        out = np.empty((s.nlogN, 8), dtype=np.float64)
        if s.nlogN:
            lib().orc_get_node_log(self.h, out.ctypes.data)
        return out

    def best_cuts(self):
        s = self.state()
        arr = (OrcCut * max(1, s.nBestCuts))()
        if s.nBestCuts:
            lib().orc_get_best_cuts(self.h, arr)
        return [(arr[i].type, arr[i].varIndex, arr[i].value) for i in range(s.nBestCuts)]


# ---------------------------------------------------------------- main.ts Solve
class OracleSolution:
    def __init__(self):
        self.feasible = True
        self.bounded = True
        self.evaluation = 0.0
        self.isIntegral = False
        self.iter = None
        self.solutionSet: dict[str, float] = {}
        self.state = None
        self.tableau: OracleTableau | None = None
        self.model: RefModel | None = None


def solve_full(jm: dict, precision=None, fast_cycles=False, pivot_log=0, node_log=0,
               max_nodes=0) -> OracleSolution:
    """Solver.Solve(model, precision, full=true) restated (main.ts:94-147, model.ts:427-449)."""
    if not jm:
        raise ValueError("Solver requires a model to operate on")
    model = RefModel(precision).loadJson(jm)
    sol = OracleSolution()
    sol.model = model
    if model.usePresolve:
        infeasible, fixed = presolve(model)
        if infeasible:  # model.ts:432-436
            sol.feasible = False
            sol.evaluation = 0.0 if model.isMinimization else -0.0
            if model.integerVariables:
                sol.iter = 0
            return sol
        for var in fixed:  # model.ts:457-461
            var.value = fixed[var]
            var.cost = 0
    M, vrow, vcol, prios, rc = model.build_tableau()
    n_idx = M.shape[0] + M.shape[1] - 2
    unres = np.zeros(n_idx, dtype=np.uint8)
    for i in model.unrestrictedVariables:
        unres[i] = 1
    ints = [v.index for v in model.integerVariables]
    tab = OracleTableau(M, vrow, vcol, precision=model.precision, unrestricted=unres, integers=ints,
                        opt_rc=rc, check_cycles=model.checkForCycles, fast_cycles=fast_cycles,
                        is_min=model.isMinimization, tolerance=model.tolerance or 0.0,
                        max_nodes=max_nodes, pivot_log=pivot_log, node_log=node_log, use_mir=bool(model.useMIRCuts))
    sol.tableau = tab
    if ints:  # tableau.ts:250-258; the service is chosen from model.options (main.ts:62-83)
        options = jm.get("options") or {}
        if options.get("useIncremental") is True:
            st = tab.incremental_branch_and_cut(options.get("nodeSelection") or "hybrid", options.get("branching") or "pseudocost")
        elif js_truthy(options.get("nodeSelection")) or js_truthy(options.get("branching")):
            st = tab.enhanced_branch_and_cut(options.get("nodeSelection") or "hybrid", options.get("branching") or "pseudocost")
        else:
            st = tab.branch_and_cut()
        sol.iter = st.bncIterations
    else:
        st = tab.simplex()
    sol.state = st
    sol.feasible = bool(st.feasible)
    sol.bounded = bool(st.bounded)
    sol.evaluation = st.evaluation if model.isMinimization else -st.evaluation
    sol.isIntegral = bool(st.isIntegral)
    # generateSolutionSet, solution.ts:35-60
    rounding = js_round(1 / model.precision)
    Mx = tab.matrix()
    vrow_f, _ = tab.maps()
    for r in range(1, st.height):
        var = model.variablesPerIndex.get(int(vrow_f[r]))
        if var is None or var.isSlack:
            continue
        sol.solutionSet[var.id] = js_round((EPSILON + Mx[r, 0]) * rounding) / rounding
    return sol


def simplify(sol: OracleSolution) -> dict:
    """buildSimplifiedResult, main.ts:173-193 (JS object key order: integer-like ids first)."""
    res: dict[str, Any] = {"feasible": sol.feasible, "result": sol.evaluation, "bounded": sol.bounded}
    if sol.isIntegral:
        res["isIntegral"] = True
    vals = {k: v for k, v in sol.solutionSet.items() if v != 0}
    ordered = {k: vals[k] for k in js_keys(vals)}
    out = {k: v for k, v in ordered.items() if k.isdigit()}
    out.update(res)
    out.update({k: v for k, v in ordered.items() if not k.isdigit()})
    return out


def Solve(jm: dict, precision=None, full=False, **kw):
    sol = solve_full(jm, precision, **kw)
    return sol if full else simplify(sol)

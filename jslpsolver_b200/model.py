"""Host-side mirror of the reference's modelling front end (Python stand-in for the unchanged
TypeScript `src/model.ts`, `src/expressions.ts`, `src/tableau/presolve.ts`).

In a Node.js deployment these files stay as they are and only `Tableau` is swapped for
`GpuTableau` (INTEGRATION.md).  This container has no Node toolchain, so the same interface is
mirrored here -- same names, argument meaning and error behaviour -- to drive the C ABI and so
that the parity tests read like the reference's own.  It produces the initial tableau
(`Tableau.setModel`, tableau.ts:382-391), which is the H2D upload source.

Data-oriented layout: constraints hold {var index -> coefficient} in insertion order and the
tableau is emitted straight into numpy arrays.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Any, Optional

import numpy as np

PRIORITY_NAMES = {"required": 0, "strong": 1, "medium": 2, "weak": 3}  # model.ts:143-161


def object_keys(obj: dict) -> list:
    """JavaScript Object.keys order: array-index-like keys ascending, then insertion order."""
    ints = [k for k in obj if isinstance(k, str) and k.isdigit() and str(int(k)) == k and int(k) < 2 ** 32 - 1]
    ints.sort(key=int)
    seen = set(ints)
    return ints + [k for k in obj if k not in seen]


def _truthy(v: Any) -> bool:
    if v is None or v is False or v == "":
        return False
    if isinstance(v, (int, float)) and not isinstance(v, bool):
        return v == v and v != 0
    return True


def math_round(x: float) -> float:
    """JavaScript Math.round (ties toward +Infinity)."""
    if x != x or x in (math.inf, -math.inf):
        return x
    lo = math.floor(x)
    return float(lo + 1) if (x - lo) >= 0.5 else float(lo)


def _div(a: float, b: float) -> float:
    try:
        return a / b
    except ZeroDivisionError:
        if a == 0 or a != a:
            return math.nan
        return math.copysign(math.inf, a) * math.copysign(1.0, b)


@dataclass(eq=False)
class Variable:  # expressions.ts:19-51
    id: str
    cost: float
    index: int
    priority: int = 0
    value: float = 0.0
    isInteger: bool = False
    isSlack: bool = False


@dataclass(eq=False)
class Term:
    variable: Variable
    coefficient: float


class Constraint:  # expressions.ts:96-203
    def __init__(self, rhs: float, isUpperBound: bool, index: int, model: "Model"):
        self.rhs = rhs
        self.isUpperBound = isUpperBound
        self.index = index
        self.model = model
        self.slack = Variable("s" + str(index), 0, index, 0, isSlack=True)
        self.coef: dict[int, Term] = {}  # var index -> term, insertion ordered
        self.relaxation: Optional[Variable] = None
        self.name: Optional[str] = None  # the JSON constraint name when loadJson built the row

    @property
    def terms(self) -> list[Term]:
        return list(self.coef.values())

    def addTerm(self, coefficient: float, variable: Variable) -> "Constraint":  # expressions.ts:119-137
        t = self.coef.get(variable.index)
        if t is None:
            self.coef[variable.index] = Term(variable, coefficient)
            self.model.updateConstraintCoefficient(self, variable, -coefficient if self.isUpperBound else coefficient)
        else:
            self.setVariableCoefficient(t.coefficient + coefficient, variable)
        return self

    def setVariableCoefficient(self, newCoefficient: float, variable: Variable) -> "Constraint":  # expressions.ts:158-184
        if variable.index == -1:
            return self
        t = self.coef.get(variable.index)
        if t is None:
            self.addTerm(newCoefficient, variable)
        elif newCoefficient != t.coefficient:
            difference = newCoefficient - t.coefficient
            if self.isUpperBound:
                difference = -difference
            t.coefficient = newCoefficient
            self.model.updateConstraintCoefficient(self, variable, difference)
        return self

    def setRightHandSide(self, newRhs: float) -> "Constraint":  # expressions.ts:144-156
        if newRhs != self.rhs:
            difference = newRhs - self.rhs
            if self.isUpperBound:
                difference = -difference
            self.rhs = newRhs
            self.model.updateRightHandSide(self, difference)
        return self

    def relax(self, weight=None, priority=None) -> None:
        self.relaxation = self.model._relaxation_variable(weight, priority)
        self._relax(self.relaxation)

    def _relax(self, rv: Optional[Variable]) -> None:
        if rv is not None:
            self.setVariableCoefficient(-1 if self.isUpperBound else 1, rv)


class Equality:  # expressions.ts:205-247
    isEquality = True

    def __init__(self, constraintUpper: Constraint, constraintLower: Constraint):
        self.upperBound, self.lowerBound = constraintUpper, constraintLower
        self.model = constraintUpper.model
        self.rhs = constraintUpper.rhs
        self.relaxation: Optional[Variable] = None

    def addTerm(self, coefficient: float, variable: Variable) -> "Equality":
        self.upperBound.addTerm(coefficient, variable)
        self.lowerBound.addTerm(coefficient, variable)
        return self

    def setRightHandSide(self, rhs: float) -> None:
        self.upperBound.setRightHandSide(rhs)
        self.lowerBound.setRightHandSide(rhs)
        self.rhs = rhs

    def relax(self, weight=None, priority=None) -> None:
        self.relaxation = self.model._relaxation_variable(weight, priority)
        for c in (self.upperBound, self.lowerBound):
            c.relaxation = self.relaxation
            c._relax(self.relaxation)


@dataclass
class PresolveResult:  # presolve.ts:16-26
    fixedVariables: dict = field(default_factory=dict)
    removedConstraints: set = field(default_factory=set)
    tightenedBounds: dict = field(default_factory=dict)
    isInfeasible: bool = False


@dataclass
class InitialTableau:
    """What Tableau.setModel produces (tableau.ts:292-391) -- the upload source."""
    matrix: np.ndarray            # H x W float64, row 0 = cost row, column 0 = RHS
    varIndexByRow: np.ndarray     # H int32
    varIndexByCol: np.ndarray     # W int32
    unrestricted: np.ndarray      # nVars uint8
    integerIndices: np.ndarray    # int32, model.integerVariables order
    optionalPriorities: list
    optionalCosts: np.ndarray     # nOpt x W float64


class Model:
    """Mirror of the reference `Model` (model.ts:24-494) for the Solve path."""

    def __init__(self, precision: Optional[float] = None, name: Optional[str] = None, branchAndCutService=None):
        from .tableau import GpuTableau  # local import: the tableau needs the CUDA library
        self.precision = 1e-8 if precision is None else precision  # tableau.ts:96
        self.name = name
        self.branchAndCutService = branchAndCutService
        self.tableau = GpuTableau(self.precision, branchAndCutService)
        self.variables: list[Variable] = []
        self.integerVariables: list[Variable] = []
        self.unrestrictedVariables: dict[int, bool] = {}
        self.constraints: list[Constraint] = []
        self.isMinimization = True
        self.tableauInitialized = False
        self.relaxationIndex = 1
        self.useMIRCuts = False
        self.checkForCycles = True
        self.messages: list = []
        self.tolerance = 0
        self.timeout = None
        self.keep_solutions = False
        self.solutions = None
        self.usePresolve = True
        self.presolveResult: Optional[PresolveResult] = None
        self.variablesPerIndex: dict[int, Variable] = {}
        self._next_index = 0

    # ------------------------------------------------------------------ builder API
    @property
    def nConstraints(self) -> int:
        return len(self.constraints)

    @property
    def nVariables(self) -> int:
        return len(self.variables)

    def _new_index(self) -> int:  # tableau.getNewElementIndex (tableau.ts:393-401): the device tableau's once it exists
        if self.tableauInitialized:
            return self.tableau.getNewElementIndex()
        i = self._next_index
        self._next_index += 1
        return i

    # ---- dynamic model modification (model.ts:196-273): edits after solve() go to the device tableau
    def updateRightHandSide(self, constraint, difference: float) -> "Model":
        if self.tableauInitialized:
            self.tableau.updateRightHandSide(constraint, difference)
        return self

    def updateConstraintCoefficient(self, constraint, variable, difference: float) -> "Model":
        if self.tableauInitialized:
            self.tableau.updateConstraintCoefficient(constraint, variable, difference)
        return self

    def setCost(self, cost: float, variable) -> "Model":
        difference = cost - variable.cost
        if not self.isMinimization:
            difference = -difference
        variable.cost = cost
        if self.tableauInitialized:
            self.tableau.updateCost(variable, difference)
        return self

    def _removeConstraint(self, constraint) -> None:
        if constraint not in self.constraints:
            return
        self.constraints.remove(constraint)
        if self.tableauInitialized:
            self.tableau.removeConstraint(constraint)
        if constraint.relaxation is not None:
            self.removeVariable(constraint.relaxation)

    def removeConstraint(self, constraint) -> "Model":
        if getattr(constraint, "isEquality", False):
            self._removeConstraint(constraint.upperBound)
            self._removeConstraint(constraint.lowerBound)
        else:
            self._removeConstraint(constraint)
        return self

    def removeVariable(self, variable) -> "Model":
        if variable not in self.variables:
            return self
        self.variables.remove(variable)
        if self.tableauInitialized:
            self.tableau.removeVariable(variable)
        return self

    def minimize(self) -> "Model":
        self.isMinimization = True
        return self

    def maximize(self) -> "Model":
        self.isMinimization = False
        return self

    def _constraint(self, rhs: float, upper: bool) -> Constraint:  # model.ts:103-124
        c = Constraint(rhs, upper, self._new_index(), self)
        self.variablesPerIndex[c.index] = c.slack
        self.constraints.append(c)
        if self.tableauInitialized:
            self.tableau.addConstraint(c)
        return c

    def smallerThan(self, rhs: float) -> Constraint:
        return self._constraint(rhs, True)

    def greaterThan(self, rhs: float) -> Constraint:
        return self._constraint(rhs, False)

    def equal(self, rhs: float) -> Equality:  # model.ts:126-134
        return Equality(self._constraint(rhs, True), self._constraint(rhs, False))

    def addVariable(self, cost=None, id=None, isInteger=False, isUnrestricted=False, priority=None) -> Variable:
        if isinstance(priority, str):
            priority = PRIORITY_NAMES.get(priority, 0)
        idx = self._new_index()
        v = Variable(id if id is not None else "v" + str(idx), 0 if cost is None else cost, idx,
                     0 if priority is None else priority, isInteger=bool(isInteger))
        if isInteger:
            self.integerVariables.append(v)
        self.variables.append(v)
        self.variablesPerIndex[idx] = v
        if isUnrestricted:
            self.unrestrictedVariables[idx] = True
        if self.tableauInitialized:  # model.ts:191-193
            self.tableau.addVariable(v)
        return v

    def _relaxation_variable(self, weight, priority) -> Optional[Variable]:  # expressions.ts:73-94
        if priority == 0 or priority == "required":
            return None
        w = 1 if weight is None else weight
        rv = self.addVariable(-w if not self.isMinimization else w, "r" + str(self.relaxationIndex), False,
                              False, 1 if priority is None else priority)
        self.relaxationIndex += 1
        return rv

    def getNumberOfIntegerVariables(self) -> int:
        return len(self.integerVariables)

    def activateMIRCuts(self, useMIRCuts: bool) -> None:
        self.useMIRCuts = useMIRCuts

    def debug(self, debugCheckForCycles: bool) -> None:
        self.checkForCycles = debugCheckForCycles

    def isFeasible(self) -> bool:
        return self.tableau.feasible

    def save(self) -> None:
        self.tableau.save()

    def restore(self) -> None:
        self.tableau.restore()

    # ------------------------------------------------------------------ loadJson (model.ts:278-419)
    def loadJson(self, jsonModel: dict) -> "Model":
        self.isMinimization = jsonModel.get("opType") != "max"
        by_min: dict[str, Constraint] = {}
        by_max: dict[str, Constraint] = {}
        cons = jsonModel["constraints"]
        for name in object_keys(cons):
            spec = cons[name] if isinstance(cons[name], dict) else {}
            weight, priority = spec.get("weight"), spec.get("priority")
            relaxed = weight is not None or priority is not None
            if spec.get("equal") is None:
                if spec.get("min") is not None:
                    c = by_min[name] = self.greaterThan(spec["min"])
                    c.name = name
                    if relaxed:
                        c.relax(weight, priority)
                if spec.get("max") is not None:
                    c = by_max[name] = self.smallerThan(spec["max"])
                    c.name = name
                    if relaxed:
                        c.relax(weight, priority)
            else:
                lo = by_min[name] = self.greaterThan(spec["equal"])
                up = by_max[name] = self.smallerThan(spec["equal"])
                lo.name = up.name = name
                if relaxed:
                    Equality(lo, up).relax(weight, priority)

        self.tolerance = jsonModel["tolerance"] if _truthy(jsonModel.get("tolerance")) else 0
        if _truthy(jsonModel.get("timeout")):
            self.timeout = jsonModel["timeout"]
        options = jsonModel.get("options")
        if _truthy(options):
            if _truthy(options.get("timeout")):
                self.timeout = options["timeout"]
            if self.tolerance == 0:
                self.tolerance = options["tolerance"] if _truthy(options.get("tolerance")) else 0
            if _truthy(options.get("useMIRCuts")):
                self.useMIRCuts = options["useMIRCuts"]
            self.checkForCycles = options["exitOnCycles"] if "exitOnCycles" in options else True
            self.keep_solutions = options["keep_solutions"] if _truthy(options.get("keep_solutions")) else False
            if options.get("presolve") is not None:
                self.usePresolve = options["presolve"]

        ints = jsonModel.get("ints") or {}
        bins = jsonModel.get("binaries") or {}
        free = jsonModel.get("unrestricted") or {}
        objective = jsonModel.get("optimize")
        variables = jsonModel["variables"]
        for vid in object_keys(variables):
            coefs = variables[vid]
            cost = coefs.get(objective) if isinstance(objective, str) else None
            is_bin = _truthy(bins.get(vid))
            var = self.addVariable(cost if _truthy(cost) else 0, vid, _truthy(ints.get(vid)) or is_bin,
                                   _truthy(free.get(vid)))
            if is_bin:
                self.smallerThan(1).addTerm(1, var)  # model.ts:392-395
            for cname in object_keys(coefs):
                if cname == objective:
                    continue
                if cname in by_min:
                    by_min[cname].addTerm(coefs[cname], var)
                if cname in by_max:
                    by_max[cname].addTerm(coefs[cname], var)
        return self

    # ------------------------------------------------------------------ Tableau.setModel source
    def initial_tableau(self) -> InitialTableau:
        nV, nC = len(self.variables), len(self.constraints)
        W, H = nV + 1, nC + 1
        M = np.zeros((H, W), dtype=np.float64)
        vrow = np.full(H, -1, dtype=np.int32)
        vcol = np.full(W, -1, dtype=np.int32)
        sign = -1.0 if self.isMinimization else 1.0
        column = {}
        optional: dict[int, np.ndarray] = {}
        for j, v in enumerate(self.variables, start=1):
            column[v.index] = j
            vcol[j] = v.index
            if v.priority == 0:
                M[0, j] = sign * v.cost
            else:  # tableau.ts:278-290
                optional.setdefault(v.priority, np.zeros(W, dtype=np.float64))[j] = sign * v.cost
        for i, c in enumerate(self.constraints, start=1):
            vrow[i] = c.index
            s = 1.0 if c.isUpperBound else -1.0  # tableau.ts:364-378
            for t in c.coef.values():
                M[i, column[t.variable.index]] = s * t.coefficient
            M[i, 0] = s * c.rhs
        unres = np.zeros(W + H - 2, dtype=np.uint8)
        for idx in self.unrestrictedVariables:
            unres[idx] = 1
        prios = sorted(optional)
        costs = np.stack([optional[p] for p in prios]) if prios else np.zeros((0, W), dtype=np.float64)
        ints = np.array([v.index for v in self.integerVariables], dtype=np.int32)
        return InitialTableau(M, vrow, vcol, unres, ints, prios, costs)

    # ------------------------------------------------------------------ solve (model.ts:427-467)
    def solve(self, *, basis=None, start=None, start_nodes: int = 1000):
        if basis is not None:  # warm start from a saved basis (DESIGN.md section 2f)
            if start is not None:
                from .mipstart import check_json
                check_json({}, basis)
            from .warmstart import solve
            return solve(self, basis)
        if start is not None:  # MIP starts (DESIGN.md section 2t)
            from .mipstart import solve
            return solve(self, start, start_nodes)
        if self.usePresolve and self.presolveResult is None:
            self.presolveResult = presolve(self)
            if self.presolveResult.isInfeasible:
                self.tableau.model = self
                self.tableau.feasible = False
                return self.tableau.getSolution()
            for variable, value in self.presolveResult.fixedVariables.items():
                variable.value = value
                variable.cost = 0  # model.ts:457-461
        if not self.tableauInitialized:
            self.tableau.setModel(self)
            self.tableauInitialized = True
        return self.tableau.solve()


# ---------------------------------------------------------------------- presolve.ts:320-492
def _get(bounds: dict, var: Variable, key: str):
    b = bounds.get(var)
    return None if b is None else b.get(key)


def presolve(model: Model) -> PresolveResult:
    res = PresolveResult()
    fixed, removed, bounds = res.fixedVariables, res.removedConstraints, res.tightenedBounds

    def set_bound(var: Variable, key: str, value: float) -> None:
        nb = dict(bounds.get(var) or {})
        nb[key] = value
        bounds[var] = nb

    def unset(x) -> bool:  # JS `!x` on a number-or-undefined
        return x is None or x == 0 or x != x

    changed, passes = True, 0
    while changed and passes < 5:
        changed = False
        passes += 1
        # singleton rows (presolve.ts:343-421)
        for con in model.constraints:
            if con in removed:
                continue
            live = [t for t in con.coef.values() if t.variable not in fixed]
            if not live:
                lhs = 0.0
                for t in con.coef.values():
                    lhs += t.coefficient * fixed[t.variable]
                ok = lhs <= con.rhs + 1e-6 if con.isUpperBound else lhs >= con.rhs - 1e-6
                if not ok:
                    res.isInfeasible = True
                    return res
                removed.add(con)
                changed = True
            elif len(live) == 1:
                var, coeff = live[0].variable, live[0].coefficient
                rhs = con.rhs
                for t in con.coef.values():
                    if t.variable is not var and t.variable in fixed:
                        rhs -= t.coefficient * fixed[t.variable]
                bound = _div(rhs, coeff)
                if con.isUpperBound:
                    key, tighter = ("upper", lambda cur: bound < cur) if coeff > 0 else ("lower", lambda cur: bound > cur)
                    cur = _get(bounds, var, key)
                    if unset(cur) or tighter(cur):
                        set_bound(var, key, bound)
                        changed = True
                removed.add(con)
        # bounds -> fixings (presolve.ts:424-467)
        for var, b in list(bounds.items()):
            if var in fixed:
                continue
            lo, up = b.get("lower"), b.get("upper")
            if lo is not None and up is not None:
                if lo > up + 1e-6:
                    res.isInfeasible = True
                    return res
                if abs(lo - up) < 1e-6:
                    fixed[var] = math_round(lo) if var.isInteger else lo
                    changed = True
            if var.isInteger and lo is not None and lo >= 0.5 and (math.inf if up is None else up) <= 1.5:
                fixed[var] = 1
                changed = True
            if var.isInteger and up is not None and up <= 0.5 and (0 if lo is None else lo) >= -0.5:
                fixed[var] = 0
                changed = True
        # activity-bound redundancy (presolve.ts:246-306)
        for con in model.constraints:
            if con in removed:
                continue
            amin = amax = 0.0
            for t in con.coef.values():
                if fixed and t.variable in fixed:
                    amin += t.coefficient * fixed[t.variable]
                    amax += t.coefficient * fixed[t.variable]
                    continue
                b = bounds.get(t.variable) if bounds else None   # one lookup per term (this loop is O(nnz) per pass)
                lo = up = None
                if b is not None:
                    lo, up = b.get("lower"), b.get("upper")
                lo = 0 if lo is None else lo
                up = 1e10 if (up is None or up == math.inf) else up
                if t.coefficient > 0:
                    amin += t.coefficient * lo
                    amax += t.coefficient * up
                else:
                    amin += t.coefficient * up
                    amax += t.coefficient * lo
            if con.isUpperBound:
                if amax <= con.rhs + 1e-6:
                    removed.add(con)
                    changed = True
                if amin > con.rhs + 1e-6:
                    res.isInfeasible = True
                    return res
            else:
                if amin >= con.rhs - 1e-6:
                    removed.add(con)
                    changed = True
                if amax < con.rhs - 1e-6:
                    res.isInfeasible = True
                    return res
        # coefficient tightening on <= rows (presolve.ts:179-240)
        for con in model.constraints:
            if con in removed or not con.isUpperBound:
                continue
            amin = 0.0
            for t in con.coef.values():
                if fixed and t.variable in fixed:
                    amin += t.coefficient * fixed[t.variable]
                    continue
                b = bounds.get(t.variable) if bounds else None
                if t.coefficient > 0:
                    lo = None if b is None else b.get("lower")
                    amin += t.coefficient * (0 if lo is None else lo)
                else:
                    up = None if b is None else b.get("upper")
                    amin += t.coefficient * (math.inf if up is None else up)
            slack = con.rhs - amin
            if slack < 0:
                continue
            for t in con.coef.values():
                v = t.variable
                if not v.isInteger or t.coefficient <= 0 or (fixed and v in fixed):
                    continue
                b = bounds.get(v) if bounds else None
                lo = up = None
                if b is not None:
                    lo, up = b.get("lower"), b.get("upper")
                lo = 0 if lo is None else lo
                up = 1 if up is None else up
                if lo >= -0.5 and up <= 1.5 and t.coefficient * (up - lo) > slack + 1e-6:
                    implied = lo + slack / t.coefficient
                    if implied < up - 1e-6:
                        cur = _get(bounds, v, "upper")
                        if unset(cur) or implied < cur:
                            set_bound(v, "upper", implied)
                            changed = True
    return res

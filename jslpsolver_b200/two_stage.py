"""Two-stage stochastic LPs: one first-stage plan for many scenarios, each with its own recourse plan.  DESIGN.md
section 2u is the contract.

The answer is an optimum of the deterministic equivalent, min c.x + sum_s p_s q_s.y_s over the first-stage rows on x and,
for every case s, the second-stage rows with case s's right-hand sides, costs and technology matrix T_s on (x, y_s), with
x, y_s >= 0 (in the model's sense; presolve is not run).  It is found by the single-cut L-shaped method in the tableau's
minimising convention: a master LP over x (the first-stage rows, the first-stage costs and the cuts so far, with a free
variable theta from the first optimality cut on) is re-solved as Solve() solves a model, and at each master plan every
case's recourse LP runs warm from one recourse tableau in one jslp_recourse_batch call, which also returns each case's
certificate row value and its cut coefficients alpha.  Everything but those two device steps is host bookkeeping, run
unchanged by the tests' CPU restatement of the device steps through `backend`."""
from __future__ import annotations

import math
from typing import Any, Optional

import numpy as np

from . import validation
from .mip_scenarios import _one_objective, _refuse
from .model import Model, _truthy, object_keys
from .scenarios import CYCLED, INFEASIBLE, OPTIMAL, UNBOUNDED, _entries, _number, edits_of

WHAT = "TwoStage()"


class Problem:
    """The model split into its stages (DESIGN.md 2u), with the cases resolved against the recourse model.

    first / second: the variable ids of each stage in the model's order; first_rows / second_rows: constraint names;
    cost: the first-stage costs in the minimising convention; tech: {second-stage constraint: [T entry per first-stage
    variable]} of the nominal model; p: the normalised probabilities."""

    def __init__(self, model: dict, first, probabilities, precision: Optional[float]):
        self.model = model
        self.objective = model["optimize"]
        self.is_min = model.get("opType") != "max"
        self.precision = Model(precision).precision
        variables, constraints = model["variables"], model.get("constraints") or {}
        names = object_keys(variables)
        if isinstance(first, str) or not isinstance(first, (list, tuple)):
            raise ValueError(f"{WHAT}: `first` is a list of variable names")
        unknown = [v for v in first if v not in variables]
        if unknown:
            raise ValueError(f"{WHAT}: `first` names unknown variable(s) {unknown}")
        chosen = set(first)
        self.first = [v for v in names if v in chosen]
        self.second = [v for v in names if v not in chosen]
        if not self.second:
            raise ValueError(f"{WHAT}: `first` names every variable: there is no second stage")
        cnames = object_keys(constraints)
        self.second_rows = [n for n in cnames if any(_coef(variables[y], n) != 0 for y in self.second)]
        srows = set(self.second_rows)
        self.first_rows = [n for n in cnames if n not in srows]
        sign = 1.0 if self.is_min else -1.0
        self.cost = [sign * _coef(variables[x], self.objective) for x in self.first]
        self.tech = {n: [float(_coef(variables[x], n)) for x in self.first] for n in self.second_rows}
        self.probabilities = probabilities

    def master_json(self, names: "Names", cuts: list) -> dict:
        """The master LP in the minimising convention: the first-stage rows and costs, then the cuts [(kind, alpha,
        rhs)] -- kind "f": alpha.x <= rhs; kind "o": theta + alpha.x >= rhs -- with theta once an optimality cut
        exists; presolve off."""
        variables, constraints = self.model["variables"], self.model.get("constraints") or {}
        cons = {n: {k: constraints[n][k] for k in ("min", "max", "equal") if constraints[n].get(k) is not None}
                for n in self.first_rows}
        out_vars = {}
        for j, x in enumerate(self.first):
            out_vars[x] = {names.objective: self.cost[j]}
            for n in self.first_rows:
                if _coef(variables[x], n) != 0:
                    out_vars[x][n] = variables[x][n]
        # theta is free: the difference of two columns >= 0.  The tableau's unrestricted-variable rule is not a
        # free-variable simplex (a master with an unrestricted theta can stop "optimal" at a point that breaks a cut)
        has_theta = any(kind == "o" for kind, _, _ in cuts)
        if has_theta:
            out_vars[names.theta + "+"] = {names.objective: 1}
            out_vars[names.theta + "-"] = {names.objective: -1}
        for k, (kind, alpha, rhs) in enumerate(cuts):
            name = names.cut(k)
            cons[name] = {"max": rhs} if kind == "f" else {"min": rhs}
            for j, x in enumerate(self.first):
                if alpha[j] != 0:
                    out_vars[x][name] = alpha[j]
            if kind == "o":
                out_vars[names.theta + "+"][name] = 1
                out_vars[names.theta + "-"][name] = -1
        return {"optimize": names.objective, "opType": "min", "constraints": cons, "variables": out_vars,
                "options": {"presolve": False}}

    def recourse_json(self, x0) -> dict:
        """The recourse LP of the nominal case at the first-stage plan x0: the second-stage rows with right-hand sides
        h - T x0 over the second-stage variables; presolve off."""
        variables, constraints = self.model["variables"], self.model["constraints"]
        cons = {}
        for n in self.second_rows:
            shift = _dot(self.tech[n], x0)
            cons[n] = {k: constraints[n][k] - shift for k in ("min", "max", "equal")
                       if constraints[n].get(k) is not None}
        out_vars = {y: {k: variables[y][k] for k in object_keys(variables[y])
                        if k == self.objective or k in cons} for y in self.second}
        options = dict(self.model.get("options") or {}, presolve=False)
        return {"optimize": self.objective, "opType": "min" if self.is_min else "max", "constraints": cons,
                "variables": out_vars, "options": options}


class Names:
    """Internal names of the master LP that no constraint, variable or attribute of the model uses."""

    def __init__(self, model: dict):
        used = set(model.get("constraints") or {}) | set(model["variables"])
        for spec in model["variables"].values():
            used |= set(spec)
        prefix = "_two_stage"
        while any(u.startswith(prefix) for u in used):
            prefix += "_"
        self.objective, self.theta, self._cut = prefix + "objective", prefix + "theta", prefix + "cut"

    def cut(self, k: int) -> str:
        return f"{self._cut}{k}"


def _coef(spec, key) -> float:
    v = spec.get(key) if isinstance(spec, dict) else None
    return v if _truthy(v) else 0


def _dot(a, x) -> float:
    """sum_j a[j] * x[j] in increasing j, unfused: the order every product with a first-stage plan uses."""
    acc = 0.0
    for aj, xj in zip(a, x):
        acc = acc + aj * xj
    return acc


def _refuse_model(model: dict) -> None:
    _refuse(model, WHAT)
    opt = model.get("optimize")
    if not isinstance(opt, (str, dict)):
        raise ValueError(f"{WHAT} takes a model with one objective")
    for key, what in (("ints", "integer"), ("binaries", "binary"), ("unrestricted", "unrestricted")):
        part = model.get(key) or {}
        if isinstance(part, dict) and any(_truthy(v) for v in part.values()):
            raise ValueError(f"{WHAT} takes a continuous model with variables >= 0: {what} variables are not "
                             "supported")


def _probabilities(probabilities, n: int) -> list:
    if probabilities is None:
        return [1.0 / n] * n
    if not isinstance(probabilities, (list, tuple)) or len(probabilities) != n:
        raise ValueError(f"{WHAT}: `probabilities` must be a list of {n} values, one per case")
    p = [_number(v, "a probability", WHAT) for v in probabilities]
    if any(v < 0 for v in p):
        raise ValueError(f"{WHAT}: probabilities must be >= 0")
    total = 0.0
    for v in p:
        total += v
    if not total > 0:
        raise ValueError(f"{WHAT}: the probabilities must have a positive sum")
    return [v / total for v in p]


class Cases:
    """Every case resolved against the recourse model m: per case, the right-hand side h of every row (m.constraints
    order), its cost edits and its technology rows.  Cases are checked here, before anything runs."""

    def __init__(self, pb: Problem, m, cases):
        self.rows = [c.index for c in m.constraints]
        self.upper = [c.isUpperBound for c in m.constraints]
        self.base = [c.rhs for c in m.constraints]
        names = [c.name for c in m.constraints]
        first_rows, second_rows = set(pb.first_rows), set(pb.second_rows)
        first_vars, fpos = set(pb.first), {x: j for j, x in enumerate(pb.first)}
        spec_of = pb.model["constraints"]
        # the model's right-hand side of every row: an equality's value for both of its rows
        nominal = [spec_of[c.name]["equal"] if spec_of[c.name].get("equal") is not None
                   else spec_of[c.name]["max" if c.isUpperBound else "min"] for c in m.constraints]
        by_name: dict = {}
        for i, c in enumerate(m.constraints):
            by_name.setdefault(c.name, []).append(i)
        self.h, self.cost_edits, self.tech = [], [], []
        per_case = False
        for k, spec in enumerate(cases):
            if not isinstance(spec, dict):
                raise ValueError(f"{WHAT}: a case is a dict with 'rhs', 'cost' and / or 'coefficients', not "
                                 f"{type(spec).__name__}")
            extra = [key for key in spec if key not in ("rhs", "cost", "coefficients")]
            if extra:
                raise ValueError(f"{WHAT}: unknown case key(s) {extra}: a case has 'rhs', 'cost' and 'coefficients'")
            for name, _ in _entries(spec, "rhs", WHAT):
                if name in first_rows:
                    raise ValueError(f"{WHAT}: case {k}: constraint {name!r} is a first-stage row: its right-hand "
                                     "side is deterministic")
            for vid, _ in _entries(spec, "cost", WHAT):
                if vid in first_vars:
                    raise ValueError(f"{WHAT}: case {k}: variable {vid!r} is first-stage: its cost is deterministic")
            # the rhs and cost entries as Solution.scenarios() checks and applies them on the recourse model
            edits = edits_of(m, {key: spec[key] for key in ("rhs", "cost") if key in spec}, WHAT)
            h = list(nominal)
            for name, value in _entries(spec, "rhs", WHAT):
                for i in by_name[name]:
                    side = "max" if m.constraints[i].isUpperBound else "min"
                    if not isinstance(value, dict):
                        h[i] = value
                    elif side in value:
                        h[i] = value[side]
            self.h.append(h)
            self.cost_edits.append([e for e in edits if e[0] == 1])
            tech = {n: list(pb.tech[n]) for n in pb.second_rows}
            for name, row in _entries(spec, "coefficients", WHAT):
                if name in first_rows:
                    raise ValueError(f"{WHAT}: case {k}: constraint {name!r} is a first-stage row: its coefficients "
                                     "are deterministic")
                if name not in second_rows:
                    raise ValueError(f"{WHAT}: case {k}: unknown constraint {name!r}")
                if not isinstance(row, dict):
                    raise ValueError(f"{WHAT}: case {k}: coefficients of {name!r} must be a dict of first-stage "
                                     f"variable -> value, not {type(row).__name__}")
                for x, v in row.items():
                    if x not in fpos:
                        what = "a second-stage variable: its coefficients are deterministic" if x in pb.model[
                            "variables"] else "not a variable of the model"
                        raise ValueError(f"{WHAT}: case {k}: coefficients of {name!r}: {x!r} is {what}")
                    tech[name][fpos[x]] = float(_number(v, f"the coefficient of {x!r} in {name!r}", WHAT))
                    per_case = True
            self.tech.append([tech[n] for n in names])
        self.per_case = per_case
        sign = np.array([1.0 if u else -1.0 for u in self.upper])
        T = np.array(self.tech, dtype=np.float64).reshape(len(cases), len(self.rows), len(pb.first))
        # the rows' tableau sign: a lower-bound row is stored negated (tableau.ts:364-378)
        signed = T * sign[None, :, None]
        self.signed = signed if per_case else signed[0]

    def edits(self, x) -> tuple:
        """(edits, offsets) of every case at the first-stage plan x: each row's right-hand side h_s - T_s x as
        Constraint.setRightHandSide passes it (skipped when unchanged), then the case's cost edits."""
        edits, offsets = [], [0]
        for s in range(len(self.h)):
            for i, label in enumerate(self.rows):
                value = self.h[s][i] - _dot(self.tech[s][i], x)
                if value != self.base[i]:
                    d = value - self.base[i]
                    edits.append((0, label, float(-d if self.upper[i] else d)))
            edits += self.cost_edits[s]
            offsets.append(len(edits))
        return edits, offsets


def run(pb: Problem, cases, backend, *, gap: float, absolute_gap: Optional[float], max_iterations: int) -> dict:
    """The L-shaped loop over a backend with master(json) -> (status, raw M[0,0], {var: value}, pivots), recourse(json)
    -> (model, pivots) (upload and solve the recourse tableau), batch(edits, offsets, rows, tech) -> the outputs of
    GpuTableau.recourse_batch, and launches() -> kernel launches so far."""
    names = Names(pb.model)
    tol_abs = pb.precision if absolute_gap is None else absolute_gap
    launches0 = backend.launches()
    p = pb.probabilities
    cuts, iterations = [], []
    lower, upper = -math.inf, math.inf
    incumbent = None
    total_pivots, recourse_lps = 0, 0
    stop, cs = None, None
    x = None
    for it in range(max_iterations):
        status, eval_raw, values, master_pivots = backend.master(pb.master_json(names, cuts))
        total_pivots += master_pivots
        if status == CYCLED:
            stop = "cycled"
            break
        if status == INFEASIBLE:
            stop, lower = "infeasible", math.inf
            break
        if status == UNBOUNDED:
            raise ValueError(f"{WHAT}: the master LP is unbounded: bound the first-stage variables, so that every "
                             "first-stage plan has a finite cost")
        x = [float(values.get(v, 0.0)) for v in pb.first]
        if any(kind == "o" for kind, _, _ in cuts):
            lower = eval_raw
        if cs is None:  # the recourse tableau, uploaded and solved once at the first master plan
            m, base_pivots = backend.recourse(pb.recourse_json(x))
            total_pivots += base_pivots
            cs = Cases(pb, m, cases)
        edits, offsets = cs.edits(x)
        out = backend.batch(edits, offsets, cs.rows, cs.signed)
        n = len(p)
        recourse_lps += n
        recourse_pivots = int(np.sum(out["p1"], dtype=np.int64) + np.sum(out["p2"], dtype=np.int64))
        total_pivots += recourse_pivots
        st = [int(v) for v in out["status"]]
        n_opt = n_feas = 0
        if any(v == CYCLED for v in st):
            stop = "cycled"
        elif any(v == INFEASIBLE for v in st):
            for s in range(n):  # one feasibility cut alpha_s . x <= beta_s per infeasible case, in case order
                if st[s] == INFEASIBLE:
                    alpha = [float(a) for a in out["alpha"][s]]
                    cuts.append(("f", alpha, float(out["cert_rhs"][s]) + _dot(alpha, x)))
                    n_feas += 1
        elif any(st[s] == UNBOUNDED and p[s] > 0 for s in range(n)):
            stop = "unbounded"
        else:
            value = _dot(pb.cost, x)
            coef, rhs = [0.0] * len(pb.first), 0.0
            for s in range(n):  # theta >= sum_s p_s (beta_s - alpha_s . x), summed in case order
                if p[s] == 0:
                    continue
                alpha = [float(a) for a in out["alpha"][s]]
                value = value + p[s] * float(out["eval_raw"][s])
                rhs = rhs + p[s] * (float(out["cert_rhs"][s]) + _dot(alpha, x))
                coef = [cj + p[s] * aj for cj, aj in zip(coef, alpha)]
            cuts.append(("o", coef, rhs))
            n_opt = 1
            if value < upper:
                upper = value
                incumbent = (list(x), {k: np.array(out[k], copy=True) for k in ("status", "eval_raw", "rhs", "vrow")})
        iterations.append({"lower": lower, "upper": upper, "optimality_cuts": n_opt, "feasibility_cuts": n_feas,
                           "recourse_pivots": recourse_pivots, "master_pivots": master_pivots})
        if stop is not None:
            break
        if upper < math.inf and upper - lower <= max(tol_abs, gap * abs(upper)):
            stop = "reached"
            break
    if stop is None:
        stop = "limit"
    sense = 1.0 if pb.is_min else -1.0
    res: dict[str, Any] = {"feasible": stop != "infeasible", "bounded": stop != "unbounded",
                           "result": None, "bound": sense * lower, "exact": stop == "reached", "first": {},
                           "cases": [], "stop": stop, "iterations": iterations, "recourse_lps": recourse_lps,
                           "pivots": total_pivots, "launches": backend.launches() - launches0}
    if stop == "unbounded":
        res["result"] = sense * -math.inf
    if incumbent is not None:
        x, out = incumbent
        res["result"] = sense * upper
        res["first"] = dict(zip(pb.first, x))
        c_x = _dot(pb.cost, x)
        label_of = {v.index: v.id for v in m.variables}
        for s in range(len(p)):
            q = float(out["eval_raw"][s])
            values = {y: 0.0 for y in pb.second}
            for r in range(1, len(out["vrow"][s])):
                vid = label_of.get(int(out["vrow"][s][r]))
                if vid is not None:
                    values[vid] = float(out["rhs"][s][r])
            res["cases"].append({"probability": p[s], "recourse": sense * q, "result": sense * (c_x + q),
                                 "values": values})
    return res


class _Device:
    """The device backend: masters through the Solve() path, the recourse tableau and its batches on the GPU."""

    def __init__(self, solver, precision):
        self.solver, self.precision, self.tab = solver, precision, None
        from .tableau import default_context
        self.context = default_context()

    def launches(self) -> int:
        return self.context.launches

    def master(self, jm):
        instance = self.solver._instance(jm, self.precision)
        instance.tableau.context = self.context
        try:
            instance.solve()
            t = instance.tableau
            st = t.lastStatus
            status = CYCLED if st.cycled else INFEASIBLE if not st.feasible else UNBOUNDED if not st.bounded else OPTIMAL
            values = {}
            rhs, _, vrow, _ = t.final_state()
            if status == OPTIMAL:
                for r in range(1, len(vrow)):
                    var = instance.variablesPerIndex.get(int(vrow[r]))
                    if var is not None and not var.isSlack:
                        values[var.id] = float(rhs[r])
            return status, float(rhs[0]) if status == OPTIMAL else math.nan, values, int(st.phase1_pivots +
                                                                                         st.phase2_pivots)
        finally:
            instance.tableau.close()

    def recourse(self, jm):
        instance = self.solver._instance(jm, self.precision)
        t = instance.tableau
        t.context = self.context
        t.setModel(instance)
        t.simplex(check_cycles=True)
        st = t.lastStatus
        if st.cycled or not st.feasible or not st.bounded:  # not optimal: the initial tableau is the start
            t.setModel(instance)
        self.tab = t
        return instance, int(st.phase1_pivots + st.phase2_pivots)

    def batch(self, edits, offsets, rows, tech):
        return self.tab.recourse_batch(edits, offsets, rows, tech)

    def close(self):
        if self.tab is not None:
            self.tab.close()


def TwoStage(solver, model: Any, cases, first, probabilities=None, *, gap=1e-9, absolute_gap=None,
             max_iterations=200, precision: Optional[float] = None, validate: bool = False, backend=None) -> dict:
    """See the module docstring.  `backend` replaces the device steps (run()'s backend; the tests' CPU restatement)."""
    if validate:
        model = validation.validate(model)
    if not model:
        raise ValueError("Solver requires a model to operate on")
    if not isinstance(model, dict):
        raise ValueError(f"{WHAT} takes a JSON model")
    _refuse_model(model)
    if not isinstance(cases, (list, tuple)) or not cases:
        raise ValueError(f"{WHAT} takes a non-empty list of cases")
    gap = _number(gap, "gap", WHAT)
    if gap < 0:
        raise ValueError(f"{WHAT}: gap must be >= 0")
    if absolute_gap is not None and _number(absolute_gap, "absolute_gap", WHAT) < 0:
        raise ValueError(f"{WHAT}: absolute_gap must be >= 0")
    if isinstance(max_iterations, bool) or not isinstance(max_iterations, int) or max_iterations < 1:
        raise ValueError(f"{WHAT}: max_iterations must be an integer >= 1")
    model = _one_objective(model)
    pb = Problem(model, first, _probabilities(probabilities, len(cases)), precision)
    # every case is checked before anything runs: against a recourse model of the same shape as the one that runs
    Cases(pb, Model(pb.precision).loadJson(pb.recourse_json([0.0] * len(pb.first))), cases)
    own = backend is None
    if own:
        backend = _Device(solver, precision)
    try:
        return run(pb, cases, backend, gap=gap, absolute_gap=absolute_gap, max_iterations=max_iterations)
    finally:
        if own:
            backend.close()

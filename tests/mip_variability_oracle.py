"""tests/mip_variability_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Variability() (DESIGN.md section 2o) restated sequentially over the C oracle: rule 1 is pool.run with k = 1 over
pool_oracle's region LPs, rule 2 the oracle's simplex of the initial tableau and near_optimal_oracle.bound, and every
node LP of rules 4 to 8 is built from the bound tableau as pool_oracle.region_lp builds a region, with the target's
cost edit (updateCost) before the cut rows, one node at a time with no batching.  The round loop is
mip_variability.run itself, so at the same width this reproduces a device run, counters included."""
from __future__ import annotations

import math

import near_optimal_oracle as NO
import pool_oracle as PO
from jslpsolver_b200 import mip_variability as MV
from jslpsolver_b200 import pool
from jslpsolver_b200.model import Model
from jslpsolver_b200.variability import _select
from oracle.ref_model import OracleTableau

OPTIMAL, INFEASIBLE, UNBOUNDED, CYCLED = PO.OPTIMAL, PO.INFEASIBLE, PO.UNBOUNDED, PO.CYCLED


def node_lp(p: PO.Problem, B, vrow_b, vcol_b, edits, cuts) -> dict:
    """One node: the bound tableau with updateCost(label, difference) for each (label, difference) of edits in order
    (a target's node has the one edit (label, -s)), the cut rows, simplex() with the cycle check on, isIntegral /
    getMostFractionalVar, and column 0 with the row labels (the outputs of PO.region_lp)."""
    o = OracleTableau(B, vrow_b, vcol_b, precision=p.m.precision, integers=p.ints, check_cycles=True)
    for label, difference in edits:
        o.update_cost(label, float(difference))
    o.add_cuts(list(cuts))
    st = o.simplex()
    status = CYCLED if st.cyclePhase else INFEASIBLE if not st.feasible else UNBOUNDED if not st.bounded else OPTIMAL
    out = {"status": status, "evaluation": float(st.evaluation) if status == OPTIMAL else
           (-math.inf if status == UNBOUNDED else 0.0), "is_integral": False, "branch_var": -1, "branch_value": 0.0,
           "pivots": int(st.lastP1 + st.lastP2), "rhs": None, "vrow": None}
    if status == OPTIMAL:
        out["is_integral"] = o.is_integral()
        if out["is_integral"]:
            out["rhs"], out["vrow"] = o.matrix()[:, 0].copy(), o.maps()[0]
        else:
            out["branch_var"], out["branch_value"] = o.most_fractional()
    return out


def region(p: PO.Problem, fixings, cuts):
    """(pool.Region, pivots) of one region of rule 1's search."""
    r = PO.region_lp(p, fixings, cuts)
    g = pool.Region(list(fixings), list(cuts))
    g.status, g.evaluation, g.integral = r["status"], r["evaluation"], bool(r["is_integral"])
    g.branch_var, g.branch_value, g.rhs, g.vrow = r["branch_var"], r["branch_value"], r["rhs"], r["vrow"]
    return g, r["pivots"]


def bound_tableau(p: PO.Problem, t: float, opt_raw: float):
    """Rule 2: (B, vrow', vcol', Delta) from the oracle's root LP optimum, its allowance t + Delta."""
    o = OracleTableau(p.M, p.vrow, p.vcol, precision=p.m.precision, integers=p.ints,
                      check_cycles=p.m.checkForCycles)
    o.simplex()
    M = o.matrix()
    vrow, vcol = o.maps()
    delta = max(0.0, float(opt_raw) - float(M[0, 0]))
    H, W = p.M.shape
    B, vrow_b, vcol_b = NO.bound(M, vrow, vcol, t + delta, NO.fresh_label(W + H - 2, W + H - 2))
    return B, vrow_b, vcol_b, delta


def variability(jm: dict, gap=0.0, absolute_gap=0.0, variables=None, constraints=None, points=False,
                max_nodes=10000, width=None, wave=1, precision=None) -> dict:
    """Variability()'s report without "launches", plus "delta" (rule 2's widening), "node_log" (the (target, cuts) of
    every node LP of rules 4 to 8 in evaluation order) and "tableau" (B, vrow', vcol')."""
    p = PO.Problem(jm, precision)
    instance = Model(precision).loadJson(jm)
    shown, rows = _select(instance, variables, constraints, MV.WHAT)
    ints = set(p.ints)
    targets = MV.targets_of(shown, rows, ints)
    pivots, log = 0, []

    def evaluate_regions(specs):
        nonlocal pivots
        out = [region(p, f, c) for f, c in specs]
        pivots += sum(n for _, n in out)
        return [g for g, _ in out]

    search = pool.Search(p.ints, p.col_of, p.binaries)
    found = pool.run(evaluate_regions, search, 1, 0.0, 0.0, max_nodes, pool.DEFAULT_WIDTH if width is None else width)
    best = MV.optimum(found, max_nodes)
    t = MV.allowance(float(gap), float(absolute_gap), float(best.rhs[0]))
    xstar = MV.plan_values(best.rhs, best.vrow)
    B, vrow_b, vcol_b, delta = bound_tableau(p, t, float(best.rhs[0]))

    def evaluate_nodes(specs):
        nonlocal pivots
        out = []
        for k, cuts in specs:
            lab, s, _ = targets[k]
            r = node_lp(p, B, vrow_b, vcol_b, [(lab, -s)], cuts)
            pivots += r["pivots"]
            log.append((k, list(cuts)))
            out.append(MV.Node(list(cuts), r["status"], r["evaluation"], r["is_integral"], r["branch_var"],
                               r["branch_value"], r["rhs"], r["vrow"]))
        return out

    out = MV.run(evaluate_nodes, targets, [xstar.get(lab, 0.0) for lab, _, _ in targets], p.m.precision, max_nodes,
                 width, wave)
    report = MV.shape(instance, shown, rows, targets, out, xstar, t, points)
    report["optimum"] = (best.evaluation if p.m.isMinimization else -best.evaluation) + 0.0
    report.update(searches=len(targets), nodes=found["nodes"] + out["nodes"], lps=found["lps"] + out["lps"],
                  rounds=found["rounds"] + out["rounds"], pivots=pivots, delta=delta, node_log=log,
                  tableau=(B, vrow_b, vcol_b))
    return report

"""tests/mip_start_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

MIP starts (DESIGN.md section 2t) restated sequentially over the C oracle: the loop of orc_branch_and_cut
(branch-and-cut.ts:54-199) written out in Python over the oracle's save / restore / addCutConstraints / simplex
primitives (apply_cuts), plus the seed stage right after the root is committed fractional.  The start nodes are
evaluated on a second oracle tableau whose root is solved and saved the same way, one node at a time, each dive to its
end before the next start's; so the main tableau's state is exactly what the loop left.  With no starts this is
orc_branch_and_cut node for node (tests/test_mip_start_cpu.py pins it); tests/test_gpu_mip_start.py checks the device
against it bit for bit."""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np

from jslpsolver_b200 import mipstart
from jslpsolver_b200.model import Model
from jslpsolver_b200.model import presolve as product_presolve
from oracle.ref_model import EPSILON, OracleTableau, RefModel, js_round, presolve, simplify, OracleSolution

SEED, FEASIBLE, INFEASIBLE, INCOMPLETE, SKIPPED = 0, 1, 2, 3, 4


def tableau(model: RefModel, max_nodes: int = 0) -> OracleTableau:
    """The oracle tableau solve_full builds for a presolved model."""
    M, vrow, vcol, _, rc = model.build_tableau()
    unres = np.zeros(M.shape[0] + M.shape[1] - 2, dtype=np.uint8)
    for i in model.unrestrictedVariables:
        unres[i] = 1
    return OracleTableau(M, vrow, vcol, precision=model.precision, unrestricted=unres,
                         integers=[v.index for v in model.integerVariables], opt_rc=rc,
                         check_cycles=model.checkForCycles, is_min=model.isMinimization,
                         tolerance=model.tolerance or 0.0, max_nodes=max_nodes, use_mir=bool(model.useMIRCuts))


def node(o: OracleTableau, cuts) -> dict:
    """applyCuts of one node (branch-and-cut.ts:33-52) and what the loop reads of it."""
    before = o.state().totalPivots
    st = o.apply_cuts(list(cuts))
    out = {"feasible": bool(st.feasible), "bounded": bool(st.bounded), "evaluation": float(st.evaluation),
           "pivots": int(st.totalPivots - before), "is_integral": False, "var": -1, "value": 0.0}
    if st.feasible:
        out["is_integral"] = o.is_integral()
        if not out["is_integral"]:
            out["var"], out["value"] = o.most_fractional()
    return out


def children(cuts, var, value):
    """branch-and-cut.ts:166-188: (high, low)."""
    high, low = [], []
    for c in cuts:
        if c[1] == var:
            (low if c[0] == 0 else high).append(c)
        else:
            high.append(c)
            low.append(c)
    return high + [(0, var, float(math.ceil(value)))], low + [(1, var, float(math.floor(value)))]


def stored(o: OracleTableau, evaluation: float):
    """What keep_solutions stores of the tableau as it stands: evaluation, column 0, row labels."""
    return evaluation, o.matrix()[:, 0].copy(), o.maps()[0].copy()


def seed_stage(model: RefModel, starts, start_nodes: int, keep_solutions: bool):
    """Every start's dive on a tableau of its own whose root is solved and saved as the loop's was.  Returns the
    status rows and the seed (index, cuts, evaluation, stored solution) or None."""
    side = tableau(model)
    node(side, [])
    side.save()
    rows, found = [], []
    for cuts in starts:
        row = {"status": INFEASIBLE, "nodes": 0, "pivots": 0, "evaluation": math.nan, "n_cuts": 0}
        stack = [list(cuts)]
        hit = None
        while True:
            if not stack:
                break
            if row["nodes"] >= start_nodes:
                row["status"] = INCOMPLETE
                break
            cl = stack.pop()
            r = node(side, cl)
            row["nodes"] += 1
            row["pivots"] += r["pivots"]
            if not r["feasible"]:
                continue
            if r["is_integral"]:
                row.update(status=FEASIBLE, evaluation=r["evaluation"], n_cuts=len(cl))
                hit = (cl, r["evaluation"])
                break
            high, low = children(cl, r["var"], r["value"])
            up = r["value"] - math.floor(r["value"]) >= 0.5
            stack += [low, high] if up else [high, low]
        rows.append(row)
        found.append(hit)
    best = None
    for i, hit in enumerate(found):
        if hit is not None and (best is None or hit[1] < found[best][1]):
            best = i
    if best is None:
        return rows, None
    rows[best]["status"] = SEED
    sol = None
    if keep_solutions:
        node(side, found[best][0])
        sol = stored(side, found[best][1])
    return rows, (best, found[best][0], found[best][1], sol)


def branch_and_cut(model: RefModel, starts=None, start_nodes: int = 1000, max_nodes: int = 0,
                   keep_solutions: bool = False) -> dict:
    """orc_branch_and_cut restated, seeded by `starts` (cut lists) when given.  Returns the final tableau `o`, the node
    log (n x 8, jslp_bnb_node_log's layout), iterations, best cuts, isIntegral, the start rows and the stored
    solutions."""
    o = tableau(model, max_nodes)
    tolerance, is_min = model.tolerance or 0.0, model.isMinimization
    heap = [(-math.inf, 0, [])]  # (relaxedEvaluation, -seq, cuts): lowest first, most recently pushed on ties
    seq = 1
    iterations, tolerance_flag, best_eval, best_cuts, is_integral = 0, True, math.inf, None, False
    log, solutions = [], []
    rows = [dict(status=SKIPPED, nodes=0, pivots=0, evaluation=math.nan, n_cuts=0) for _ in (starts or [])]
    early = False
    while heap and tolerance_flag:
        if max_nodes > 0 and iterations >= max_nodes:
            break
        bpe = o.state().bestPossibleEval
        threshold = bpe * (1 + tolerance) if is_min else bpe * (1 - tolerance)
        if tolerance > 0 and best_eval < threshold:
            tolerance_flag = False
        top = min(heap)
        heap.remove(top)
        relaxed, _, cuts = top
        if relaxed > best_eval:
            continue
        r = node(o, cuts)
        iterations += 1
        nl = [iterations, len(cuts), float(r["feasible"]), r["evaluation"], -1, -1, 0, r["pivots"]]
        log.append(nl)
        if not r["feasible"] or r["evaluation"] > best_eval or r["evaluation"] == best_eval:
            continue  # no optional objectives: an equal value is never better
        if r["is_integral"]:
            nl[4] = 1
            is_integral = True
            if iterations == 1:
                early = True
                break
            best_eval, best_cuts = r["evaluation"], cuts
            if keep_solutions:
                solutions.append(stored(o, r["evaluation"]))
            continue
        nl[4], nl[5], nl[6] = 0, r["var"], r["value"]
        if iterations == 1:
            o.save()
        high, low = children(cuts, r["var"], r["value"])
        heap.append((r["evaluation"], -seq, high))
        heap.append((r["evaluation"], -seq - 1, low))
        seq += 2
        if iterations == 1 and starts and r["bounded"]:
            rows, seed = seed_stage(model, starts, start_nodes, keep_solutions)
            if seed is not None:
                best_eval, best_cuts, is_integral = seed[2], seed[1], True
                if keep_solutions:
                    solutions.append(seed[3])
    if best_cuts is not None and not early:
        node(o, best_cuts)
    return {"o": o, "node_log": np.array(log, dtype=np.float64).reshape(-1, 8), "iterations": iterations,
            "best_cuts": [] if best_cuts is None or early else list(best_cuts), "is_integral": is_integral,
            "starts": rows, "solutions": solutions}


def solve(jm: dict, start=None, start_nodes: int = 1000, max_nodes: int = 0, precision=None):
    """Solve(jm, start=..., full=True) restated: (simplified result, mipStart report, branch_and_cut's dict or None)."""
    m = Model(precision).loadJson(jm)  # the product's mapping of names to cut lists (no GPU needed)
    plan_list = mipstart.plans(start) if start is not None else []
    m.presolveResult = product_presolve(m) if m.usePresolve else None
    model = RefModel(precision).loadJson(jm)
    sol = OracleSolution()
    if model.usePresolve:
        infeasible, fixed = presolve(model)
        if infeasible:
            sol.feasible = False
            sol.evaluation = 0.0 if model.isMinimization else -0.0
            mapped = mipstart.cut_lists(m, plan_list)
            return simplify(sol), mipstart.report(m, mapped, [], math.inf), None
        for var in fixed:
            var.value = fixed[var]
            var.cost = 0
    mapped = mipstart.cut_lists(m, plan_list)
    starts = [s["cuts"] for s in mapped if s["cuts"] is not None]
    res = branch_and_cut(model, starts if start is not None else None, start_nodes, max_nodes,
                         bool(model.keep_solutions))
    o = res["o"]
    st = o.state()
    sol.feasible, sol.bounded = bool(st.feasible), bool(st.bounded)
    sol.evaluation = st.evaluation if model.isMinimization else -st.evaluation
    sol.isIntegral = res["is_integral"]
    rounding = js_round(1 / model.precision)
    Mx, (vrow, _) = o.matrix(), o.maps()
    for r in range(1, st.height):
        var = model.variablesPerIndex.get(int(vrow[r]))
        if var is not None and not var.isSlack:
            sol.solutionSet[var.id] = js_round((EPSILON + Mx[r, 0]) * rounding) / rounding
    native = [SimpleNamespace(**row) for row in res["starts"]]
    return simplify(sol), mipstart.report(m, mapped, native, st.evaluation), res

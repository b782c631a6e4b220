"""tests/repair_mip_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

RepairMIP() (DESIGN.md section 2r) restated sequentially over the C oracle: the elastic tableau E is
repair_oracle.elastic of the model's initial tableau (rule 1), every node LP is lexicographic_mip_oracle.Level's
node_lp on a stage's tableau with the node's cut rows, one node at a time with no batching, each stage's search is
lexicographic_mip.search itself (rules 2 and 3), R_1 is lexicographic_oracle.solve of E and stage 2's tableau is
lexicographic_oracle.child of it (rule 3).  At the same width this reproduces a device run, counters included."""
from __future__ import annotations

import numpy as np

import lexicographic_mip_oracle as LMO
import lexicographic_oracle as LO
import near_optimal_oracle as NO
import pool_oracle as PO
import repair_oracle as RO
from jslpsolver_b200 import lexicographic_mip as LM
from jslpsolver_b200 import mip_variability as MV
from jslpsolver_b200.repair_mip import WHAT, stage_entry
from oracle.sensitivity import json_row_names

OPTIMAL, CYCLED = PO.OPTIMAL, PO.CYCLED


def _stage(level: LMO.Level, entry: dict, log: list, P, max_nodes, width, wave) -> dict:
    """One stage's search on level, its node pivots and counters in entry; log gets every node's cuts in order."""
    def evaluate(specs):
        nodes = []
        for _, cuts in specs:
            node, pivots = level.node(cuts)
            entry["pivots"] += pivots
            log.append(list(cuts))
            nodes.append(node)
        return nodes

    H, W = level.T.shape
    found = LM.search(evaluate, P, max_nodes, width, wave(H, W) if callable(wave) else wave)
    entry.update(nodes=found["nodes"], lps=found["lps"], rounds=found["rounds"])
    return found


def repair_mip(jm, weights=None, objective=True, gap=0.0, absolute_gap=0.0, max_nodes=10000, width=None, wave=1,
               precision=None):
    """(RepairMIP()'s result without "launches", details).  `wave(height, width)` (or a number) stands for the
    default width's wave of a stage tableau.  details = {"rows", "weights", "E": (E, vrow, vcol), "levels": the
    stages' Levels (None for a face that keeps only column 0), "node_log": per stage, "delta": Delta or None}."""
    opt = jm.get("optimize")
    if isinstance(opt, dict):
        key = list(opt)[0]
        jm = dict(jm, optimize=key, opType="max" if opt[key] == "max" else "min")
    p = PO.Problem(jm, precision)
    model, P = p.m, p.m.precision
    H, W = p.M.shape
    if weights is None:  # every row, the `x <= 1` rows of binaries (after the JSON rows) included
        rows, w = list(range(1, len(model.constraints) + 1)), [1.0] * len(model.constraints)
    else:
        rows, w = RO.row_weights(jm, weights)
    label = H + W - 2
    n = label + len(rows)
    E, vr, vc, crashed = RO.elastic(p.M, p.vrow, p.vcol, P, rows, w, label)
    key = jm.get("optimize") if isinstance(jm.get("optimize"), str) else None
    sense = "min" if model.isMinimization else "max"
    out = {"feasible": True, "violation": None, "constraints": [], "values": None, "result": None,
           "stop": "reached", "stages": [], "pivots": 0}
    stages = out["stages"]
    level = LMO.Level(E, vr, vc, n, p)
    det = {"rows": rows, "weights": w, "E": (E, vr, vc), "levels": [level], "node_log": [[]], "delta": None}
    s1 = dict(stage_entry("violation"), crashed=len(crashed), width=E.shape[1], height=H)
    stages.append(s1)
    found = _stage(level, s1, det["node_log"][0], P, max_nodes, width, wave)
    state, plan = found["state"], found["witness"]
    assert state != "unbounded", "the violation came out unbounded"
    if state == "cycled":
        out["stop"], plan = "cycled", None
    elif state == "limit":
        if plan is None:
            raise ValueError(f"{WHAT}: the search of stage 1 hit max_nodes={max_nodes} before any integer plan; "
                             "raise max_nodes")
        s1["exact"], s1["bound"] = False, found["bound"] + 0.0
        out["stop"] = "limit"
    elif plan is None:
        out["feasible"], out["stop"] = False, "infeasible"
    if plan is not None:
        vstar = s1["optimum"] = float(plan.rhs[0]) + 0.0
    if plan is not None and objective and state == "exact":
        t = max(float(absolute_gap), float(gap) * abs(vstar))
        root = LO.solve(E, vr, vc, P)
        s1["pivots"] += root[1] + root[2]
        if root[0] == CYCLED:
            out["stop"] = "cycled"
        else:
            assert root[0] == OPTIMAL, root[0]
            d = det["delta"] = max(0.0, float(plan.rhs[0]) - float(root[3][0, 0]))
            arg = t + d
            s2 = dict(stage_entry("face" if arg == 0.0 else "bound"), allowance=t)
            stages.append(s2)
            cost = np.zeros(n)
            cost[np.asarray(p.vcol[1:], dtype=np.int64)] = p.M[0, 1:]
            T, vrt, vct, _ = LO.child(root[3], root[4], root[5], P, cost, arg, NO.fresh_label(n, n))
            stage2 = None if T is None else LMO.Level(T, vrt, vct, n + (1 if arg > 0.0 else 0), p)
            det["levels"].append(stage2)
            det["node_log"].append([])
            if stage2 is None:
                s2["optimum"] = RO.sum_objective(model, jm, key, _plan(model, plan)[0])
            else:
                s2.update(width=T.shape[1], height=T.shape[0])
                found = _stage(stage2, s2, det["node_log"][1], P, max_nodes, width, wave)
                state, best = found["state"], found["witness"]
                if state in ("unbounded", "cycled"):
                    out["stop"] = state
                else:
                    assert best is not None or state == "limit", "stage 2 lost the plan of stage 1"
                    if state == "limit":
                        s2["exact"], s2["bound"] = False, LM.signed(sense, found["bound"])
                        out["stop"] = "limit"
                    if best is not None:
                        plan = best
                        s2["optimum"] = LM.signed(sense, float(best.rhs[0]))
                    else:
                        s2["optimum"] = RO.sum_objective(model, jm, key, _plan(model, plan)[0])
    if plan is not None:
        x, at = _plan(model, plan)
        e = [at.get(label + j, 0.0) for j in range(len(rows))]
        det["e"] = e
        violation = 0.0
        for wj, ej in zip(w, e):
            violation += wj * ej
        out["violation"] = violation
        names = json_row_names(jm)
        for r, wj, ej in zip(rows, w, e):
            if ej > P:
                con = model.constraints[r - 1]
                name = names[r - 1] if r <= len(names) else con.index  # a binary's row has no name
                out["constraints"].append({"name": name, "type": "max" if con.isUpperBound else "min",
                                           "rhs": con.rhs, "weight": wj, "violation": ej,
                                           "repairedRhs": con.rhs + ej if con.isUpperBound else con.rhs - ej})
        out["values"] = dict(zip([v.id for v in model.variables], x))
        out["result"] = RO.sum_objective(model, jm, key, x)
    for name in ("nodes", "lps", "rounds", "pivots"):
        out[name] = sum(s[name] for s in stages)
    return out, det


def _plan(model, node) -> tuple:
    at = MV.plan_values(node.rhs, node.vrow)
    return tuple(at.get(v.index, 0.0) for v in model.variables), at

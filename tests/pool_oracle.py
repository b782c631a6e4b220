"""The solution-pool search of DESIGN.md section 2m, restated literally and sequentially over the C oracle: every
region is built from the model's initial tableau in numpy (fixings) and the oracle (cut rows, simplex, integrality
scan), one region at a time, with no batching and no speculation.  tests/test_pool_cpu.py checks it against brute
force; tests/test_gpu_pool.py checks Pool() and jslp_pool_batch against it."""
from __future__ import annotations

import math

import numpy as np

from oracle.ref_model import EPSILON, OracleTableau, RefModel, js_round, js_truthy

OPTIMAL, INFEASIBLE, UNBOUNDED, CYCLED = 0, 1, 2, 3


class Problem:
    """The model as the search sees it: initial tableau, integer labels in integerIndices order, their columns and the
    binaries."""

    def __init__(self, jm: dict, precision=None):
        self.jm = jm
        self.m = RefModel(precision).loadJson(jm)
        self.M, self.vrow, self.vcol, _, _ = self.m.build_tableau()
        self.ints = [v.index for v in self.m.integerVariables]
        self.col_of = {int(self.vcol[c]): c for c in range(1, len(self.vcol))}
        bins = jm.get("binaries") or {}
        self.binaries = {v.index for v in self.m.variables if js_truthy(bins.get(v.id))}


def region_lp(p: Problem, fixings, cuts) -> dict:
    """One region: fixings applied to a copy of the initial tableau in list order, cut rows appended, simplex(),
    isIntegral / getMostFractionalVar, and column 0 with the row labels."""
    M = p.M.copy()
    for col, v in fixings:
        M[:, 0] = M[:, 0] - v * M[:, col]  # two roundings, no FMA: edit_axpy_sub
        M[:, col] = 0.0
    o = OracleTableau(M, p.vrow, p.vcol, precision=p.m.precision, integers=p.ints, check_cycles=p.m.checkForCycles)
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


def assignment(p: Problem, fixings, res) -> dict:
    """{label: integer} of an integral region: basic integer variables rounded, fixed ones at their fixing, the rest
    non-basic at 0."""
    z = {lab: 0 for lab in p.ints}
    for r in range(1, len(res["vrow"])):
        if int(res["vrow"][r]) in z:
            z[int(res["vrow"][r])] = int(math.floor(float(res["rhs"][r]) + 0.5))
    for col, v in fixings:
        z[int(p.vcol[col])] = int(v)
    return z


def children(p: Problem, fixings, cuts, res) -> list:
    """The regions that replace a popped one, in push order."""
    if not res["is_integral"]:
        # branch-and-cut.ts:155-190: a cut on the branching variable goes to cutsLow when it is a `min` cut and to
        # cutsHigh when it is a `max` cut; every other cut goes to both; then the new cut of each child
        var, value = res["branch_var"], res["branch_value"]
        high, low = [], []
        for c in cuts:
            if c[1] == var:
                if c[0] == 0:
                    low.append(c)
                else:
                    high.append(c)
            else:
                high.append(c)
                low.append(c)
        high.append((0, var, float(math.ceil(value))))
        low.append((1, var, float(math.floor(value))))
        return [(list(fixings), high), (list(fixings), low)]
    # the region minus z: child m fixes the free integer variables before j_m at z, then excludes z at j_m with a `max`
    # cut at z - 1 (none when z = 0) and a `min` cut at z + 1 (none for a binary at 1); a new cut replaces the cuts of
    # its type on its variable, and a variable that becomes fixed loses its cuts
    z = assignment(p, fixings, res)
    fixed = {int(p.vcol[col]) for col, _ in fixings}
    fx, cs, out = list(fixings), list(cuts), []
    for lab in p.ints:
        if lab in fixed:
            continue
        if z[lab] != 0:
            out.append((list(fx), [c for c in cs if not (c[1] == lab and c[0] == 1)] + [(1, lab, float(z[lab] - 1))]))
        if not (lab in p.binaries and z[lab] == 1):
            out.append((list(fx), [c for c in cs if not (c[1] == lab and c[0] == 0)] + [(0, lab, float(z[lab] + 1))]))
        fx.append((p.col_of[lab], float(z[lab])))
        cs = [c for c in cs if c[1] != lab]
    return out


def pool(jm: dict, k: int = 10, gap: float = 0.0, absolute_gap: float = 0.0, max_nodes: int = 100000,
         precision=None) -> dict:
    """The sequential search.  Returns {"solutions": [{"evaluation", "z", "values", "result", "rank"}], "stop",
    "nodes", "allowance"} with Pool()'s meanings ("nodes" = region LPs solved)."""
    p = Problem(jm, precision)
    heap = []  # [evaluation, -seq, fixings, cuts, res]: lowest evaluation first, most recently pushed on ties
    seq = 0
    sols, stop, t = [], None, None
    root = region_lp(p, [], [])
    nodes = 1
    if root["status"] == UNBOUNDED:
        stop = "unbounded"
    elif root["status"] == OPTIMAL:
        heap.append((root["evaluation"], -seq, [], [], root))
        seq += 1
    while stop is None:
        if not heap:
            stop = "exhausted"
            break
        top = min(heap, key=lambda e: (e[0], e[1]))
        if sols and top[0] > sols[0]["evaluation"] + t:
            stop = "gap"
            break
        if nodes >= max_nodes:
            stop = "limit"
            break
        heap.remove(top)
        ev, _, fixings, cuts, res = top
        if res["is_integral"]:
            sols.append({"evaluation": ev, "z": assignment(p, fixings, res), "fixings": fixings, "res": res})
            if len(sols) == 1:
                t = max(absolute_gap, gap * abs(ev))
            if len(sols) == k:
                stop = "k"
                break
        kids = [(f, c, region_lp(p, f, c)) for f, c in children(p, fixings, cuts, res)]
        nodes += len(kids)
        if any(r["status"] == UNBOUNDED for _, _, r in kids):
            stop = "unbounded"
            break
        for f, c, r in kids:
            if r["status"] == OPTIMAL:
                heap.append((r["evaluation"], -seq, f, c, r))
                seq += 1
    rounding = js_round(1 / p.m.precision)
    out = []
    for rank, s in enumerate(sols, start=1):
        row_of = {int(s["res"]["vrow"][r]): r for r in range(1, len(s["res"]["vrow"]))}
        values = {}
        for v in p.m.variables:
            if v.index in s["z"]:
                values[v.id] = float(s["z"][v.index])
            elif v.index in row_of:
                values[v.id] = js_round((EPSILON + float(s["res"]["rhs"][row_of[v.index]])) * rounding) / rounding
            else:
                values[v.id] = 0.0
        out.append({"evaluation": s["evaluation"], "z": s["z"], "values": values, "rank": rank,
                    "result": (s["evaluation"] if p.m.isMinimization else -s["evaluation"]) + 0.0})
    return {"solutions": out, "stop": stop, "nodes": nodes, "allowance": t}

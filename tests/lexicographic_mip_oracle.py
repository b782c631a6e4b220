"""tests/lexicographic_mip_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

LexicographicMIP() (DESIGN.md section 2q) restated sequentially over the C oracle: the level tableaux are
lexicographic_oracle.child of the root LP optimum lexicographic_oracle.solve gives (rule 1), every node LP is
mip_variability_oracle.node_lp on the level's tableau with no edits and the node's cut rows, one node at a time with no
batching, and each level's search is lexicographic_mip.search itself (rule 2), so at the same width this reproduces a
device run, counters included.

A face drops columns, so its labels have gaps the oracle's label tables do not allow.  Every level tableau is handed
to the oracle with its labels renamed to their rank (order kept, so the integrality scan visits the integer labels in
the same order) and every label read back is named back; a cut row's label, past the ranks, is named after the
device's next free label of that level."""
from __future__ import annotations

import math
import types

import numpy as np

import lexicographic_oracle as LO
import mip_variability_oracle as MVO
import near_optimal_oracle as NO
import pool_oracle as PO
from jslpsolver_b200 import lexicographic_mip as LM
from jslpsolver_b200 import mip_variability as MV
from jslpsolver_b200.model import object_keys
from oracle import frontier as OF

OPTIMAL, INFEASIBLE, UNBOUNDED, CYCLED = PO.OPTIMAL, PO.INFEASIBLE, PO.UNBOUNDED, PO.CYCLED


class Level:
    """A level tableau T (original labels vrow / vcol) whose next free label on the device is `n`, with the renaming
    the oracle runs it under."""

    def __init__(self, T, vrow, vcol, n: int, p: PO.Problem):
        self.T, self.vrow, self.vcol, self.n = np.asarray(T, dtype=np.float64), vrow, vcol, int(n)
        self.present = sorted([int(v) for v in vrow[1:]] + [int(v) for v in vcol[1:]])
        self.rank = {v: k for k, v in enumerate(self.present)}
        self.ren = types.SimpleNamespace(m=p.m, ints=[self.rank[v] for v in p.ints if v in self.rank])
        self.vrow_r = np.array([-1] + [self.rank[int(v)] for v in vrow[1:]], dtype=np.int32)
        self.vcol_r = np.array([-1] + [self.rank[int(v)] for v in vcol[1:]], dtype=np.int32)

    def back(self, lab: int) -> int:
        lab = int(lab)
        return self.present[lab] if lab < len(self.present) else self.n + lab - len(self.present)

    def node(self, cuts) -> tuple:
        """(MV.Node, pivots) of the node with these cut rows."""
        r = MVO.node_lp(self.ren, self.T, self.vrow_r, self.vcol_r, [],
                        [(t, self.rank[int(v)], x) for t, v, x in cuts])
        bvar = self.back(r["branch_var"]) if r["branch_var"] >= 0 else r["branch_var"]
        vrow = None if r["vrow"] is None else np.array([-1] + [self.back(v) for v in r["vrow"][1:]], dtype=np.int32)
        return MV.Node(list(cuts), r["status"], r["evaluation"], r["is_integral"], bvar, r["branch_value"], r["rhs"],
                       vrow), r["pivots"]


def chain(jm: dict, gap=0.0, absolute_gap=0.0, max_nodes=10000, width=None, wave=1, precision=None):
    """(LexicographicMIP()'s result without "launches", details) where details[k] = {"level": Level or None,
    "node_log": [cuts of every node LP in evaluation order], "delta": Delta_k or None}."""
    opt = jm["optimize"]
    keys = object_keys(opt)
    senses = {k: "max" if opt[k] == "max" else "min" for k in keys}
    g, a = LO.gaps(gap, keys), LO.gaps(absolute_gap, keys)
    working = dict(jm, optimize=keys[0], opType=senses[keys[0]])
    p = PO.Problem(working, precision)
    model, P = p.m, p.m.precision
    H, W = p.M.shape
    cur = Level(p.M, p.vrow, p.vcol, W + H - 2, p)
    levels, det = [], []
    out = {"feasible": True, "bounded": True, "stop": "reached", "objectives": None, "values": None, "levels": levels}
    plan, arg = None, 0.0
    for k, key in enumerate(keys):
        lv = LM.level_entry(key, senses[key])
        levels.append(lv)
        d = {"level": None, "node_log": [], "delta": None}
        det.append(d)
        if k > 0 and cur is not None:
            cost = np.zeros(cur.n)
            c = OF.cost2(model, working, key, senses[key], {})
            cost[:len(c)] = c
            T, vr, vc, _ = LO.child(root[3], root[4], root[5], P, cost, arg, NO.fresh_label(cur.n, cur.n))
            cur = None if T is None else Level(T, vr, vc, cur.n + (1 if arg > 0.0 else 0), p)
        d["level"] = cur
        if cur is None:
            lv["optimum"] = LO.sum_objective(model, working, key, plan)
        else:
            lv.update(kind="initial" if k == 0 else "face" if arg == 0.0 else "bound", width=cur.T.shape[1],
                      height=cur.T.shape[0])

            def evaluate(specs, cur=cur, lv=lv, d=d):
                nodes = []
                for _, cuts in specs:
                    node, pivots = cur.node(cuts)
                    lv["pivots"] += pivots
                    d["node_log"].append(list(cuts))
                    nodes.append(node)
                return nodes

            found = LM.search(evaluate, P, max_nodes, width, wave)
            lv.update(nodes=found["nodes"], lps=found["lps"], rounds=found["rounds"])
            state, best = found["state"], found["witness"]
            if state in ("unbounded", "cycled"):
                out["stop"] = state
                break
            if state == "limit":
                if best is None and plan is None:
                    raise ValueError(f"{LM.WHAT}: the search of level 1 ({key!r}) hit max_nodes={max_nodes} before "
                                     "any integer plan; raise max_nodes")
                lv["exact"], lv["bound"] = False, LM.signed(senses[key], found["bound"])
            if best is None and state == "exact":
                assert k == 0, "a later level lost the plan of the level before it"
                out["feasible"], out["stop"] = False, None
                break
            if best is not None:
                at = MV.plan_values(best.rhs, best.vrow)
                plan = tuple(at.get(v.index, 0.0) for v in model.variables)
                lv["optimum"] = LM.signed(senses[key], float(best.rhs[0]))
            else:
                lv["optimum"] = LO.sum_objective(model, working, key, plan)
            if state == "limit":
                out["stop"] = "limit"
                break
        if k + 1 < len(keys):
            t = max(a[k], g[k] * abs(lv["optimum"]))
            assert not math.isinf(t)
            lv["allowance"] = t
            if cur is not None:
                root = LO.solve(cur.T, cur.vrow, cur.vcol, P)
                lv["pivots"] += root[1] + root[2]
                if root[0] == CYCLED:
                    out["stop"] = "cycled"
                    break
                assert root[0] == OPTIMAL, root[0]
                d["delta"] = max(0.0, float(best.rhs[0]) - float(root[3][0, 0]))
                arg = t + d["delta"]
    if out["stop"] == "unbounded":
        out["bounded"] = False
    if plan is not None:
        out["values"] = {v.id: x for v, x in zip(model.variables, plan)}
        out["objectives"] = {key: LO.sum_objective(model, working, key, plan) for key in keys}
    for name in ("nodes", "lps", "rounds", "pivots"):
        out[name] = sum(lv[name] for lv in levels)
    return out, det

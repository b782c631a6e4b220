"""tests/frontier_mip_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

FrontierMIP() (DESIGN.md section 2s) restated sequentially over the C oracle: the ends are lexicographic_mip_oracle.chain
of the two orders of the objectives (rule 1), every box search's node LP is box_node_lp on the box tableau -- the
oracle's updateRightHandSide and updateCost edits in order, the node's cut rows, simplex() with the cycle check on, one
node at a time with no batching -- and the stage and box loops are mip_variability.run and frontier_mip.trace
themselves, so at the same width this reproduces a device run, counters included."""
from __future__ import annotations

import math

import lexicographic_mip_oracle as LMO
import pool_oracle as PO
from jslpsolver_b200 import frontier_mip as FM
from jslpsolver_b200 import lexicographic_mip as LM
from jslpsolver_b200 import mip_variability as MV
from jslpsolver_b200 import pool
from jslpsolver_b200.model import Model
from oracle.ref_model import OracleTableau

OPTIMAL, INFEASIBLE, UNBOUNDED, CYCLED = PO.OPTIMAL, PO.INFEASIBLE, PO.UNBOUNDED, PO.CYCLED


def box_node_lp(p: PO.Problem, edits, cuts, tableau=None) -> dict:
    """One node of jslp_box_batch: the snapshot (M, vrow, vcol) = tableau, by default the initial tableau of p, with
    edits [(kind, label, difference), ...] applied in order (kind 0 updateRightHandSide, kind 1 updateCost), the cut
    rows, simplex() with the cycle check on, isIntegral / getMostFractionalVar, and column 0 with the row labels when
    integral (the outputs of MVO.node_lp)."""
    M, vrow, vcol = (p.M, p.vrow, p.vcol) if tableau is None else tableau
    o = OracleTableau(M, vrow, vcol, precision=p.m.precision, integers=p.ints, check_cycles=True)
    for kind, label, difference in edits:
        if kind == 0:
            o.update_rhs(label, float(difference))
        else:
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


def _chain(jm: dict, max_nodes, width, wave):
    """lexicographic_mip_oracle.chain at gap 0 with each level's wave taken from its tableau's shape, as
    lexicographic_mip.run_stage takes it on the device."""
    search = LM.search

    def shaped(evaluate, P, max_nodes, width, _):
        h, w = evaluate.__defaults__[0].T.shape  # the level the restatement's evaluate closes over
        return search(evaluate, P, max_nodes, width, wave(h, w))

    LMO.LM.search = shaped
    try:
        return LMO.chain(jm, max_nodes=max_nodes, width=width)
    finally:
        LMO.LM.search = search


def frontier_mip(jm: dict, step=None, max_points=1000, max_nodes=10000, width=None, wave=lambda h, w: 1,
                 precision=None):
    """(FrontierMIP()'s result without "launches", details) where details = {"node_log": [(target edits, cuts) of
    every box node LP in evaluation order], "stages": [live boxes of every stage]}.  wave(height, width) is the default
    width's wave of a tableau of that shape (with the 8-level dive)."""
    keys, senses = FM.objectives(jm)
    step, proven = FM.step_of(jm, keys, step)
    max_points = pool._count("max_points", max_points, 2, FM.WHAT)
    max_nodes = pool._count("max_nodes", max_nodes, 1, FM.WHAT)
    width = None if width is None else pool._count("width", width, 1, FM.WHAT)
    loaded = FM.loads(jm, keys, senses)
    o1, o2, r1, r2 = loaded["names"]
    count = {"searches": 0, "nodes": 0, "lps": 0, "rounds": 0, "pivots": 0}
    det = {"node_log": [], "stages": []}

    def extreme(which: str, order):
        m = Model(precision).loadJson(loaded[which])
        sense = {o1: senses[keys[0]], o2: senses[keys[1]]}
        try:
            out, _ = _chain(dict(loaded[which], optimize={k: sense[k] for k in order}), max_nodes, width, wave)
        except ValueError as e:
            raise ValueError(FM.no_plan(keys[0 if which == "first" else 1], max_nodes)) from e
        count["searches"] += sum(1 for lv in out["levels"] if lv["kind"] is not None)
        for name in ("nodes", "lps", "rounds", "pivots"):
            count[name] += out[name]
        plan = None
        if out["stop"] == "reached":
            plan = FM.point(m, jm, keys, senses, tuple(out["values"][v.id] for v in m.variables))
        return out, plan

    ra, a = extreme("first", [o1, o2])
    if not ra["feasible"]:
        return dict(FM.result(keys, senses, step, proven, [], None, None, 0.0), feasible=False, exact=True,
                    **count), det
    rb, b = extreme("second", [o2, o1])
    assert rb["feasible"]
    p = PO.Problem(loaded["box"], precision)
    P = p.m.precision
    stop = FM.ends_stop(ra, rb)
    if stop is not None or FM.same_image(a, b, P):
        return dict(FM.result(keys, senses, step, proven, [a, b], None, stop or "reached", P), **count), det
    bm = Model(precision).loadJson(loaded["box"])  # the labels and variables of the box tableau
    slack, cost = FM.box_edits(bm, jm, keys, senses, (r1, r2))
    H, W = p.M.shape

    def stage(specs):
        det["stages"].append(len(specs))
        edits = [FM.node_spec(slack, cost, u1, u2, k) for u1, u2, k in specs]

        def evaluate(nodes):
            out = []
            for k, cuts in nodes:
                r = box_node_lp(p, edits[k], cuts)
                count["pivots"] += r["pivots"]
                det["node_log"].append((edits[k], list(cuts)))
                out.append(MV.Node(list(cuts), r["status"], r["evaluation"], r["is_integral"], r["branch_var"],
                                   r["branch_value"], r["rhs"], r["vrow"]))
            return out

        n = len(specs)
        out = MV.run(evaluate, [LM.OWN] * n, [math.inf] * n, P, max_nodes, width, wave(H, W), shared=False)
        for name in ("nodes", "lps", "rounds"):
            count[name] += out[name]
        return [(state, None if w is None or state != "exact" else FM.point(bm, jm, keys, senses, FM.plan_of(bm, w)))
                for state, w in zip(out["state"], out["witness"])]

    traced = FM.trace(a, b, step, P, max_points, stage)
    count["searches"] += traced["searches"]
    return dict(FM.result(keys, senses, step, proven, [a, b], traced, traced["stop"], P), **count), det

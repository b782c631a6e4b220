"""The MIP conflict of DESIGN.md section 2n, restated literally and sequentially over the C oracle: every node LP is
built from the model's initial tableau (the kept rows, relabelled densely as oracle/iis.py does) and the oracle (cut
rows, phase 1, integrality scan), one node at a time, each test a plain depth-first search, each filter the
one-at-a-time deletion filter.  tests/test_conflict_cpu.py checks it against SciPy's HiGHS and drives the host search
of jslpsolver_b200/conflict.py with node(); tests/test_gpu_conflict.py checks Conflict() and jslp_conflict_batch
against it."""
from __future__ import annotations

import math

import numpy as np

from oracle import iis as oracle_iis
from oracle.ref_model import OracleTableau, RefModel

FEASIBLE, INFEASIBLE, UNDECIDED = 0, 1, 2  # test verdicts; a node's status uses 2 for "cycled"


class Problem:
    """The model as the tests see it: initial tableau, unrestricted flags, integer labels in integerIndices order, and
    the first label a cut row takes (the whole tableau's element count)."""

    def __init__(self, jm: dict, precision=None):
        self.jm = jm
        self.m = RefModel(precision).loadJson(jm)
        self.M, self.vrow, self.vcol, _, _ = self.m.build_tableau()
        H, W = self.M.shape
        self.unres = np.zeros(H + W - 2, dtype=np.uint8)
        for i in self.m.unrestrictedVariables:
            self.unres[i] = 1
        self.ints = [v.index for v in self.m.integerVariables]
        self.rows = list(range(1, H))
        self.first_index = H + W - 2
        self.precision = self.m.precision


def node(p: Problem, rows, J, cuts) -> dict:
    """One node LP: rows 0 + `rows` of the initial tableau, the cut rows, phase 1 (cycle check on), and the integrality
    scan over the labels J (in integerIndices order, so positions and ties agree with the whole list's).  Labels are in
    the original numbering, cut rows from p.first_index."""
    keep = [0] + sorted(rows)
    labels = sorted(set(int(v) for v in p.vrow[keep[1:]]) | set(int(v) for v in p.vcol[1:]))
    new = {old: i for i, old in enumerate(labels)}
    vr = np.array([-1] + [new[int(p.vrow[r])] for r in keep[1:]], dtype=np.int32)
    vc = np.array([-1] + [new[int(v)] for v in p.vcol[1:]], dtype=np.int32)
    u = np.array([p.unres[old] for old in labels], dtype=np.uint8)
    tab = OracleTableau(np.ascontiguousarray(p.M[keep]), vr, vc, precision=p.precision, unrestricted=u,
                        integers=[new[j] for j in J], check_cycles=True, fast_cycles=True)
    tab.add_cuts([(t, new[v], val) for t, v, val in cuts])
    pivots = int(tab.phase1())
    st = tab.state()
    status = UNDECIDED if st.cyclePhase == 1 else FEASIBLE if st.feasible else INFEASIBLE

    def back(v):
        v = int(v)
        return -1 if v < 0 else labels[v] if v < len(labels) else p.first_index + v - len(labels)

    out = {"status": status, "pivots": pivots, "is_integral": False, "branch_var": -1, "branch_value": 0.0,
           "rhs": tab.matrix()[:, 0].copy(), "vrow": np.array([back(v) for v in tab.maps()[0]], dtype=np.int64)}
    if status == FEASIBLE:
        out["is_integral"] = tab.is_integral()
        if not out["is_integral"]:
            v, x = tab.most_fractional()
            out["branch_var"], out["branch_value"] = back(v), x
    return out


def replace(cuts, cut):
    """cuts without those of cut's type on cut's variable, then cut (branch-and-cut.ts:166-179)."""
    return [c for c in cuts if not (c[0] == cut[0] and c[1] == cut[1])] + [cut]


def test(p: Problem, rows, J, max_nodes: int):
    """(verdict, witness node or None, nodes evaluated) of test(rows, J): depth-first, last pushed popped first; a
    fractional node pushes its `min ceil` child, then its `max floor` child."""
    stack, nodes, cycled = [[]], 0, False
    while stack:
        cuts = stack.pop()
        r = node(p, rows, J, cuts)
        nodes += 1
        if r["status"] == UNDECIDED:
            cycled = True
        elif r["status"] == FEASIBLE:
            if r["is_integral"]:
                return FEASIBLE, r, nodes
            v, x = r["branch_var"], r["branch_value"]
            stack.append(replace(cuts, (0, v, float(math.ceil(x)))))
            stack.append(replace(cuts, (1, v, float(math.floor(x)))))
        if stack and nodes >= max_nodes:
            return UNDECIDED, None, nodes
    return (UNDECIDED if cycled else INFEASIBLE), None, nodes


def conflict(jm: dict, max_nodes: int = 10000, precision=None) -> dict:
    """The start, the row filter and the integrality filter, literally.  Returns {"verdict"} of the whole model when it
    is not INFEASIBLE; otherwise {"verdict", "relaxation", "rows", "ints", "irreducible", "row_witness",
    "int_witness", "problem"} with the witnesses by member."""
    p = Problem(jm, precision)
    rows, ints = p.rows, p.ints
    v, _, _ = test(p, rows, ints, max_nodes)
    if v != INFEASIBLE:
        return {"verdict": v}
    _, support, relaxation = oracle_iis.start_set(p.M, p.vrow, p.vcol, p.unres, p.precision)
    S0 = rows
    if relaxation == INFEASIBLE and support != rows and test(p, support, ints, max_nodes)[0] == INFEASIBLE:
        S0 = support
    B, irreducible, row_witness = list(S0), True, {}
    for s in list(S0):
        v, w, _ = test(p, [x for x in B if x != s], ints, max_nodes)
        if v == INFEASIBLE:
            B.remove(s)
        else:
            row_witness[s] = w
            irreducible &= v == FEASIBLE
    J, int_witness = [], {}
    if test(p, B, [], max_nodes)[0] != INFEASIBLE:
        J = list(ints)
        for j in ints:
            v, w, _ = test(p, B, [x for x in J if x != j], max_nodes)
            if v == INFEASIBLE:
                J.remove(j)
            else:
                int_witness[j] = w
                irreducible &= v == FEASIBLE
    return {"verdict": INFEASIBLE, "relaxation": relaxation, "rows": B, "ints": J, "irreducible": irreducible,
            "row_witness": row_witness, "int_witness": int_witness, "problem": p}


def plan(w, ids: dict):
    """{"values": {id: value}} of a witness node, as Conflict() reports it."""
    if w is None:
        return None
    at = {int(w["vrow"][r]): float(w["rhs"][r]) for r in range(1, len(w["vrow"]))}
    return {"values": {vid: at.get(lab, 0.0) for lab, vid in ids.items()}}


def row_owners(jm: dict) -> list:
    """For every tableau row 1.. in order: (constraint name, None) for the rows loadJson builds from `constraints`
    (min before max, an equality as both), then (None, variable id) for the `x <= 1` row of each binary."""
    from oracle.ref_model import js_keys, js_truthy
    out = []
    for name in js_keys(jm["constraints"]):
        spec = jm["constraints"][name] if isinstance(jm["constraints"][name], dict) else {}
        if spec.get("equal") is not None:
            out += [(name, None), (name, None)]
        else:
            out += [(name, None)] * ((spec.get("min") is not None) + (spec.get("max") is not None))
    bins = jm.get("binaries") or {}
    return out + [(None, vid) for vid in js_keys(jm["variables"]) if js_truthy(bins.get(vid))]


def named(res: dict) -> dict:
    """The fields of Conflict()'s result that do not count work, from conflict()."""
    p = res["problem"]
    ids = {v.index: v.id for v in p.m.variables}
    owners = row_owners(p.jm)
    constraints, bounds, names = [], [], []
    for r in res["rows"]:
        con = p.m.constraints[r - 1]
        w = plan(res["row_witness"].get(r), ids)
        name, vid = owners[r - 1]
        if name is None:
            bounds.append({"variable": vid, "type": "max", "rhs": 1, "witness": w})
            continue
        constraints.append({"name": name, "type": "max" if con.isUpperBound else "min", "rhs": con.rhs, "witness": w})
        if name not in names:
            names.append(name)
    return {"constraints": constraints, "bounds": bounds,
            "integers": [{"variable": ids[j], "witness": plan(res["int_witness"].get(j), ids)} for j in res["ints"]],
            "names": names, "relaxation": {INFEASIBLE: "infeasible", FEASIBLE: "feasible"}.get(res["relaxation"],
                                                                                             "undecided"),
            "irreducible": res["irreducible"]}

"""Integer models whose root LP is clean and one of whose later node LPs cycles (tests/test_cycle_models_cpu.py checks
them on the oracle, tests/test_gpu_cycle_nodes.py runs them on the device; not a test module).

Every node of branch and cut restores the root's optimal tableau, adds its cut rows and runs phase 1 and phase 2, each
with a fresh history of (leaving, entering) pairs; the reference stops an LP before it repeats a block of pairs and
reports the node infeasible.  A witness is a root optimum from which one added bound row sends the node LP into a
repeat.  Both builders hide a cycling block behind an integer y that the root sets to 1/2 through the row
`Y: y + ... <= 1/2` with a large cost on y, so that the low child `y <= 0` is the node that cycles:

* phase 1 (`phase1_witness`): the rows hold the negative transpose of Beale's tableau, so phase 1 (a dual simplex:
  the most negative right-hand side leaves, the largest quotient -cost / coefficient enters, the lowest column on a
  tie) walks Beale's cycle on the dual side.  The rows that Beale's positive reduced costs make negative carry
  `-2 y`, so at the root, where y = 1/2, they are feasible and the LP ends after two pivots.  In the child the
  cut row's only negative entry is Y's slack; pivoting it in sets y = 0 and the negative rows reappear.
* phase 2 (`phase2_witness`): Beale's LP itself.  Y also holds `eps * x` on Beale's two columns with negative cost,
  with eps = 2^-27 below the precision 1e-8 and K * eps = 8 at least their reduced costs: at the root y enters, and
  the one pivot leaves every reduced cost <= 0.  The child's cut row repeats Y's entries negated; phase 1 ignores
  the -eps entries (not below -precision), pivots Y's slack in on the cut row, and so adds K * eps back to the
  reduced costs: phase 2 then starts from Beale's own row 0 over the untouched degenerate rows and cycles.

Beale's cycle is exact in dyadic arithmetic and never ends without the check; these blocks are Beale's with some rows
and columns scaled by factors like 1.1 and 2/3 (found by a seeded search on the oracle), which still cycle under the
reference's rules with a cycle of length 6, chosen so that the rounding of a full turn breaks a tie in a later turn: without the check the LP leaves the cycle by
itself after a few turns (tens of pivots).  So the shared-memory node kernel, which runs a node LP to its end and
screens the log afterwards, ends such a node well inside its 512-entry log and reaches its cycle-hit redo, not the
overflow redo.

pad > 0 adds that many continuous columns p_k (cost 1, never entering) in rows `p_k <= 3` (never binding): a tableau
past one SM's shared memory whose nodes run in node slots, with the pivots of the small model."""
import numpy as np

EPS = 2.0 ** -27
# Beale's tableau: rows r1..r3 over x4..x7 and the costs (min)
BEALE_ROWS = {"r1": [0.25, -8, -1, 9], "r2": [0.5, -12, -0.5, 3], "r3": [0, 0, 1, 0]}
BEALE_COST = [-0.75, 20, -0.5, 6]
PAD = 300
# node-slot step counts at which a node's repeat spans several host polls (the default, 32, sees it in one)
SPANNING_STEPS = (1, 2, 3)


def _pad(jm: dict, pad: int) -> dict:
    for k in range(pad):
        jm["constraints"][f"p{k}"] = {"max": 3}
        jm["variables"][f"p{k}"] = {"cost": 1, f"p{k}": 1}
    if pad:
        jm["name"] += f"_pad{pad}"
    return jm


def phase1_witness(pad: int = 0, prune: bool = False) -> dict:
    """Phase 1 cycles in node 2 (y <= 0).  Rows d4..d7 are Beale's columns x4..x7 negated and transposed, row d_j
    scaled by 1.1, 1.1, 0.1, 2/3 and the columns u0..u2 (Beale's rows) by 1, 2/3, 7; cost 3 on u2 (Beale's right-hand
    side 1); y costs -10 and carries -2 in d4 and d6.

    prune adds a plan and an order: Y gains -w (cost 12, so y >= 1 is feasible at a cost of 1 over the root), and an
    integer z (first, so the root branches on it: both are 1/2) with p >= z - 1/2 (cost 1) and q >= 1/2 - z (cost 4).
    The child z >= 1 (value -4.5) is better than z <= 0 (value -3): its y >= 1 child is an integer plan of value -3.5
    that pops before (z <= 0, y <= 0), whose relaxed value -3 is worse, so the reference never evaluates that cycling
    node; the device speculates it in the same round."""
    base = {"d4": [-0.25, -0.5, 0, -0.75], "d5": [8, 12, 0, 20], "d6": [1, 0.5, -1, -0.5], "d7": [-9, -3, 0, 6]}
    fr = {"d4": 1.1, "d5": 1.1, "d6": 0.1, "d7": 2 / 3}
    fc = (1, 2 / 3, 7)
    g = {"d4": -2, "d6": -2}
    rows = {}
    for j, row in base.items():
        rows[j] = [v * fr[j] for v in row[:3]] + [row[3] * fr[j]]
        for i in range(3):
            rows[j][i] *= fc[i]
    cons = {j: {"max": r[3]} for j, r in rows.items()}
    cons["Y"] = {"max": 0.5}
    var = {f"u{i}": {"cost": (0, 0, 3)[i], **{j: r[i] for j, r in rows.items() if r[i]}} for i in range(3)}
    if prune:
        cons["Zp"] = {"max": 0.5}
        cons["Zq"] = {"max": -0.5}
        var["z"] = {"Zp": 1, "Zq": -1}
        var["p"] = {"cost": 1, "Zp": -1}
        var["q"] = {"cost": 4, "Zq": -1}
        var["w"] = {"cost": 12, "Y": -1}
    var["y"] = {"cost": -10, "Y": 1, **g}
    jm = {"name": "CyclePhase1" + ("Prune" if prune else ""), "optimize": "cost", "opType": "min", "constraints": cons,
          "variables": var, "ints": {"z": 1, "y": 1} if prune else {"y": 1}, "options": {"presolve": False}}
    return _pad(jm, pad)


def phase2_witness(pad: int = 0) -> dict:
    """Phase 2 cycles in node 2 (y <= 0): Beale's rows r1..r3 scaled by 1, 1.3, 3 and its columns x0..x3 by 2/3, 1,
    1, 1.1 (costs included); Y: y + eps x0 + eps x2 <= 1/2 with y's cost -2^30."""
    fr = (1, 1.3, 3)
    fc = (2 / 3, 1, 1, 1.1)
    rows = {r: [v * fr[k] for v in row] for k, (r, row) in enumerate(BEALE_ROWS.items())}
    cost = [c * fc[j] for j, c in enumerate(BEALE_COST)]
    for r in rows:
        rows[r] = [v * fc[j] for j, v in enumerate(rows[r])]
    var = {f"x{j}": {"cost": cost[j], **{r: v[j] for r, v in rows.items() if v[j]}} for j in range(4)}
    var["x0"]["Y"] = EPS
    var["x2"]["Y"] = EPS
    var["y"] = {"cost": -2.0 ** 30, "Y": 1}
    jm = {"name": "CyclePhase2", "optimize": "cost", "opType": "min", "variables": var,
          "constraints": {"r1": {"max": 0}, "r2": {"max": 0}, "r3": {"max": 1}, "Y": {"max": 0.5}},
          "ints": {"y": 1}, "options": {"presolve": False}}
    return _pad(jm, pad)


# (id, model, {1-based committed node: (phase, cycle length, phase-1 pivots, phase-2 pivots)}); the prune models also
# speculate the cycling node (z <= 0, y <= 0), which the reference never commits
PHASE1_CYCLE = {2: (1, 6, 12, 0)}
PHASE2_CYCLE = {2: (2, 6, 1, 11)}
PRUNE_CYCLE = {4: (1, 6, 14, 0)}


def cases() -> list:
    return [("phase1", phase1_witness(), PHASE1_CYCLE), ("phase1_padded", phase1_witness(PAD), PHASE1_CYCLE),
            ("phase2", phase2_witness(), PHASE2_CYCLE), ("phase2_padded", phase2_witness(PAD), PHASE2_CYCLE),
            ("prune", phase1_witness(prune=True), PRUNE_CYCLE),
            ("prune_padded", phase1_witness(PAD, prune=True), PRUNE_CYCLE)]


def node_cuts(jm: dict, max_nodes: int = 0) -> list:
    """The cut list of every committed node, in commit order, by replaying the reference's loop on the node log: the
    root pushes its children (high, then low) with its evaluation, best-first pops the smallest relaxed value, the
    most recently pushed first on ties, and a node whose relaxed value exceeds the incumbent's is skipped."""
    from oracle import ref_model
    sol = ref_model.solve_full(jm, fast_cycles=True, node_log=1 << 20, max_nodes=max_nodes)
    nl = sol.tableau.node_log()
    heap, seq, out, best = [(-np.inf, 0, [])], 0, [], np.inf
    for row in nl:
        while True:
            heap.sort(key=lambda e: (e[0], -e[1]))
            rel, _, cuts = heap.pop(0)
            if rel <= best:
                break
        out.append(cuts)
        feasible, ev, integral, var, val = row[2], row[3], row[4], int(row[5]), row[6]
        if not feasible or ev > best:
            continue
        if integral == 1:
            best = ev
            continue
        # branch-and-cut.ts: an earlier bound on the branching variable goes to the child it does not contradict
        seq += 1
        heap.append((ev, seq, [c for c in cuts if not (c[1] == var and c[0] == 0)] + [(0, var, float(np.ceil(val)))]))
        seq += 1
        heap.append((ev, seq, [c for c in cuts if not (c[1] == var and c[0] == 1)] + [(1, var, float(np.floor(val)))]))
    return out


def replay(jm: dict, cuts: list, check_cycles: bool = True, pivot_limit: int = 0):
    """One node LP on the oracle as branch and cut runs it: the root solved and saved, then the cut list applied.
    Returns the oracle tableau (state(), pivot_log())."""
    from oracle import ref_model
    m = ref_model.RefModel().loadJson(jm)
    M, vrow, vcol, _, _ = m.build_tableau()
    t = ref_model.OracleTableau(M, vrow, vcol, integers=[v.index for v in m.integerVariables],
                                check_cycles=check_cycles, fast_cycles=True, pivot_log=1 << 16)
    t.simplex()
    t.save()
    if pivot_limit:
        t.set_pivot_limit(pivot_limit)
    t.apply_cuts(cuts)
    return t

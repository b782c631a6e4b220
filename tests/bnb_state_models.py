"""Branch-and-cut models whose node logs carry infeasible nodes between feasible ones (tests/test_bnb_state_cpu.py checks
them on the oracle, tests/test_gpu_bnb_state.py runs them on the device; not a test module).

An infeasible node's log row holds the evaluation the tableau had before its LP (the last committed node that set
one), so these models are where a node LP that writes the tableau's evaluation out of commit order shows up in column 3
of the node log and in the result of Solve()."""
import numpy as np

# Speculation widths of the device modes that evaluate more than one node per round.
WIDTHS = (2, 4, 8, 16, 32)


def leak_model(high_fractional: bool = False) -> dict:
    """min x (+ z) over x - y >= 0.5, x integer: the root gives x = 0.5, its low child x <= 0 is infeasible and pops
    before its high child x >= 1 (equal relaxed values, the later push first).  With high_fractional a second integer z
    (2 z - x >= 0.5, min x + z) makes the root branch on z, and the high child z >= 1 is fractional again (1.75).
    Two variables in every row keep presolve from turning the rows into bounds."""
    if not high_fractional:
        return {"name": "LeakMIP", "optimize": "v", "opType": "min", "constraints": {"c": {"min": 0.5}},
                "variables": {"x": {"v": 1, "c": 1}, "y": {"c": -1}}, "ints": {"x": 1}}
    return {"name": "LeakMIPFractional", "optimize": "v", "opType": "min",
            "constraints": {"c": {"min": 0.5}, "d": {"min": 0.5}},
            "variables": {"x": {"v": 1, "c": 1, "d": -1}, "y": {"c": -1}, "z": {"v": 1, "d": 2}},
            "ints": {"x": 1, "z": 1}}


def parity_mip(n: int, seed: int, ub: int = 3, pad: int = 0) -> dict:
    """sum 2 x_i = 2 k + 1 with integer 0 <= x_i <= ub and random costs: the LP relaxation is feasible, no integer plan
    exists, so every branch ends in an infeasible node.  pad > 0 adds that many integer columns y_j (positive cost,
    zero at every node) with a row y_j + x_(j mod n) <= ub + 2 each, presolve off: a tableau of n + pad + 1 columns and
    n + pad + 1 rows whose nodes do not fit shared memory."""
    rng = np.random.default_rng(seed)
    k = int(rng.integers(1, n * ub // 2))
    cost = rng.integers(1, 20, n) + rng.random(n).round(2)
    cons = {"odd": {"equal": 2 * k + 1}}
    variables = {f"x{i}": {"cost": float(cost[i]), "odd": 2, f"u{i}": 1} for i in range(n)}
    for i in range(n):
        cons[f"u{i}"] = {"max": ub}
    for j in range(pad):
        cons[f"p{j}"] = {"max": ub + 2}
        variables[f"x{j % n}"][f"p{j}"] = 1
        variables[f"y{j}"] = {"cost": float(1 + j % 7), f"p{j}": 1}
    jm = {"name": f"ParityMIP_{n}_{seed}_{pad}", "optimize": "cost", "opType": "min", "constraints": cons,
          "variables": variables, "ints": {v: 1 for v in variables}}
    if pad:
        jm["options"] = {"presolve": False}
    return jm


def root_infeasible_mip() -> dict:
    """An integer model whose root LP is infeasible after phase-1 pivots (presolve off, so branch and cut sees it)."""
    return {"name": "RootInfeasibleMIP", "optimize": "v", "opType": "max",
            "constraints": {"a": {"min": 4}, "b": {"min": 3}, "s": {"max": 5}},
            "variables": {"x": {"v": 1, "a": 1, "s": 1}, "y": {"v": 2, "b": 1, "s": 1}, "z": {"v": 1, "a": 1, "b": -1}},
            "ints": {"x": 1, "y": 1}, "options": {"presolve": False}}


# (id, model, max_nodes caps to run it at; 0 = no cap)
SMALL_PARITY = parity_mip(4, 0)          # the whole tree: 167 nodes
CAPPED_PARITY = parity_mip(6, 0)         # 2003 nodes uncapped; run capped only
PADDED_PARITY = parity_mip(6, 0, pad=300)


def leaks(node_log: np.ndarray, width: int) -> list:
    """Rows i of a node log (0-based) that are infeasible and whose column 3 differs from that of a feasible row within
    the next width - 1 commits: a round of `width` nodes that wrote a later node's evaluation into the tableau before
    row i was committed would change row i."""
    out = []
    for i in range(len(node_log)):
        if node_log[i, 2] != 0:
            continue
        nxt = node_log[i + 1:i + width]
        if any(r[2] != 0 and r[3] != node_log[i, 3] for r in nxt):
            out.append(i)
    return out


def stop_caps(node_log: np.ndarray, width: int = 4, n: int = 3) -> list:
    """max_nodes values at which the loop stops right after committing an infeasible node that leaks() flags at
    `width`: the first n of them."""
    return [i + 1 for i in leaks(node_log, width)[:n]]


def cases() -> list:
    """Every model of the device file with the caps it runs at."""
    from oracle import ref_model
    full = ref_model.solve_full(CAPPED_PARITY, fast_cycles=True, node_log=1 << 20, max_nodes=2003).tableau.node_log()
    capped = sorted(set(stop_caps(full, 4) + stop_caps(full, 8)[-1:] + [97]))
    return ([("leak", leak_model(), (0, 2)), ("leak_fractional", leak_model(True), (0, 2, 3)),
             ("parity_small", SMALL_PARITY, (0,)), ("root_infeasible", root_infeasible_mip(), (0,))]
            + [("parity_capped", CAPPED_PARITY, tuple(capped)), ("parity_padded", PADDED_PARITY, (60,))])

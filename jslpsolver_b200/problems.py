"""Synthetic workloads for BASELINE.json's configs (SURVEY.md 8d "Concrete inputs").

Distributions follow the reference's seeded generators (src/test-utils/problem-generator.ts:
generateResourceAllocation 297-340, generateKnapsack); the random stream itself is numpy's
(the reference's Mulberry32 accumulates its seed as a double and is not reproducible across
languages for millions of draws -- SURVEY.md 8c), so one materialised instance is fed to every
implementation that is compared.
"""
from __future__ import annotations

import numpy as np

from .model import InitialTableau


def dense_packing_lp_arrays(n_vars: int, n_cons: int, seed: int = 12345):
    """max c.x  s.t.  A x <= b, x >= 0 with a_ij ~ U{1..20}, b_i ~ U{100..500}, c_j ~ U{1..50}."""
    rng = np.random.default_rng(seed)
    A = rng.integers(1, 21, size=(n_cons, n_vars)).astype(np.float64)
    b = rng.integers(100, 501, size=n_cons).astype(np.float64)
    c = rng.integers(1, 51, size=n_vars).astype(np.float64)
    return A, b, c


def dense_packing_lp_tableau(n_vars: int, n_cons: int, seed: int = 12345) -> InitialTableau:
    """The tableau `Model.loadJson(dense_packing_lp_model(...))` + `Tableau.setModel` would build
    (tableau.ts:319-380), emitted directly: constraints take element indices 0..m-1, variables
    m..m+n-1 (model.ts:288-332,382-416); opType max -> cost row +c (tableau.ts:332-339)."""
    A, b, c = dense_packing_lp_arrays(n_vars, n_cons, seed)
    H, W = n_cons + 1, n_vars + 1
    M = np.zeros((H, W), dtype=np.float64)
    M[0, 1:] = c
    M[1:, 0] = b
    M[1:, 1:] = A
    vrow = np.concatenate([[-1], np.arange(n_cons)]).astype(np.int32)
    vcol = np.concatenate([[-1], n_cons + np.arange(n_vars)]).astype(np.int32)
    return InitialTableau(M, vrow, vcol, np.zeros(W + H - 2, dtype=np.uint8), np.zeros(0, dtype=np.int32), [],
                          np.zeros((0, W), dtype=np.float64))


def lp_model(A, b, c, lower=None, maximize: bool = True) -> dict:
    """A dense LP as a jsLPSolver JSON model: row i is `min: b_i` where lower[i] is set, `max: b_i` otherwise.  Every
    entry of A except +0.0 becomes a term (so -0.0 survives as an explicit coefficient)."""
    A, b, c = np.asarray(A, dtype=np.float64), np.asarray(b, dtype=np.float64), np.asarray(c, dtype=np.float64)
    lower = np.zeros(len(b), dtype=bool) if lower is None else np.asarray(lower, dtype=bool)
    present = (A != 0) | np.signbit(A) | np.isnan(A)
    constraints = {f"c{i}": {"min" if lower[i] else "max": float(b[i])} for i in range(len(b))}
    variables = {}
    for j in range(A.shape[1]):
        v = {"objective": float(c[j])}
        for i in np.nonzero(present[:, j])[0]:
            v[f"c{i}"] = float(A[i, j])
        variables[f"x{j}"] = v
    return {"name": f"LP_{A.shape[1]}x{A.shape[0]}", "optimize": "objective", "opType": "max" if maximize else "min",
            "constraints": constraints, "variables": variables}


def lp_tableau(A, b, c, lower=None, maximize: bool = True) -> InitialTableau:
    """The tableau `Model.loadJson(lp_model(A, b, c, lower, maximize)).initial_tableau()` builds, emitted directly (for
    shapes where the JSON front end is slow): a `min` row is stored negated (tableau.ts:364-378), an absent term stays
    +0.0, and a falsy cost enters as 0 times the objective's sign."""
    A, b, c = np.asarray(A, dtype=np.float64), np.asarray(b, dtype=np.float64), np.asarray(c, dtype=np.float64)
    n_cons, n_vars = A.shape
    lower = np.zeros(n_cons, dtype=bool) if lower is None else np.asarray(lower, dtype=bool)
    present = (A != 0) | np.signbit(A) | np.isnan(A)
    s = np.where(lower, -1.0, 1.0)
    sign = 1.0 if maximize else -1.0
    H, W = n_cons + 1, n_vars + 1
    M = np.zeros((H, W), dtype=np.float64)
    M[0, 1:] = sign * np.where((c != 0) & ~np.isnan(c), c, 0.0)
    M[1:, 0] = s * b
    M[1:, 1:] = np.where(present, s[:, None] * A, 0.0)
    vrow = np.concatenate([[-1], np.arange(n_cons)]).astype(np.int32)
    vcol = np.concatenate([[-1], n_cons + np.arange(n_vars)]).astype(np.int32)
    return InitialTableau(M, vrow, vcol, np.zeros(W + H - 2, dtype=np.uint8), np.zeros(0, dtype=np.int32), [],
                          np.zeros((0, W), dtype=np.float64))


def dense_packing_lp_model(n_vars: int, n_cons: int, seed: int = 12345) -> dict:
    """Same instance as a jsLPSolver JSON model (use for moderate sizes)."""
    A, b, c = dense_packing_lp_arrays(n_vars, n_cons, seed)
    constraints = {f"resource{i}": {"max": float(b[i])} for i in range(n_cons)}
    variables = {}
    for j in range(n_vars):
        v = {"profit": float(c[j])}
        for i in range(n_cons):
            v[f"resource{i}"] = float(A[i, j])
        variables[f"activity{j}"] = v
    return {"name": f"DensePacking_{n_vars}x{n_cons}_seed{seed}", "optimize": "profit", "opType": "max",
            "constraints": constraints, "variables": variables}


def alternative_optima_arrays(n_vars: int, n_cons: int, seed: int = 12345, dup: int = 3, par: int = 3):
    """(A, b, c) of a packing LP `max c.x, A x <= b, x >= 0` whose optimum is not unique (dual degeneracy planted two
    ways).  The first n_vars - dup - par columns and n_cons - 1 rows are dense_packing_lp_arrays' distributions, with
    the costs of the first `dup` columns raised by 50 so that they tend to be basic; the next `dup` columns repeat
    those columns and costs exactly (a copy of a basic variable has reduced cost 0).  The last `par` variables appear
    only in the last row, `blend`, with entries a_j ~ U{1..20} and costs exactly 3 a_j: the objective is parallel to
    that row over them, the row binds, and all but one of them are non-basic at reduced cost 0."""
    base = n_vars - dup - par
    assert dup >= 0 and par >= 0 and base >= dup and n_cons >= 2
    rng = np.random.default_rng(seed)
    A = np.zeros((n_cons, n_vars), dtype=np.float64)
    A[:n_cons - 1, :base] = rng.integers(1, 21, size=(n_cons - 1, base))
    b = rng.integers(100, 501, size=n_cons).astype(np.float64)
    c = np.zeros(n_vars, dtype=np.float64)
    c[:base] = rng.integers(1, 51, size=base)
    c[:dup] += 50.0
    A[:, base:base + dup] = A[:, :dup]
    c[base:base + dup] = c[:dup]
    A[n_cons - 1, base + dup:] = rng.integers(1, 21, size=par)
    c[base + dup:] = 3.0 * A[n_cons - 1, base + dup:]
    return A, b, c


def alternative_optima_model(n_vars: int, n_cons: int, seed: int = 12345, dup: int = 3, par: int = 3) -> dict:
    """alternative_optima_arrays as a jsLPSolver JSON model (lp_model's names: x0.., c0..)."""
    m = lp_model(*alternative_optima_arrays(n_vars, n_cons, seed, dup, par))
    m["name"] = f"AlternativeOptima_{n_vars}x{n_cons}_seed{seed}"
    return m


def alternative_optima_multi_model(n_vars: int, n_cons: int, n_objectives: int, seed: int = 12345, dup: int = 3,
                                   par: int = 3) -> dict:
    """alternative_optima_model with `optimize` = {objective: max, obj1: min, obj2: max, ...} (the extra senses
    alternate, starting with min).  The extra attributes are U{0..20} per variable from a generator seeded with (seed,
    n_objectives); the `dup` copies take their originals' values, so every objective keeps each copy tied with its
    original and a face at allowance 0 is not a single point."""
    m = alternative_optima_model(n_vars, n_cons, seed, dup, par)
    m["name"] = f"AlternativeOptima{n_objectives}obj_{n_vars}x{n_cons}_seed{seed}"
    base = n_vars - dup - par
    rng = np.random.default_rng((seed, n_objectives))
    extra = rng.integers(0, 21, size=(n_objectives - 1, n_vars)).astype(np.float64)
    extra[:, base:base + dup] = extra[:, :dup]
    m["optimize"] = {"objective": "max", **{f"obj{k}": "min" if k % 2 else "max" for k in range(1, n_objectives)}}
    for j, v in enumerate(m["variables"].values()):
        for k in range(1, n_objectives):
            v[f"obj{k}"] = float(extra[k - 1, j])
    return m


def dense_packing_multi_model(n_vars: int, n_cons: int, n_objectives: int, seed: int = 12345) -> dict:
    """dense_packing_lp_model with `optimize` = {profit: max, attr1: max, ...}: the extra objective attributes are
    U{1..50} per variable, drawn from the same seed after the packing instance."""
    rng = np.random.default_rng(seed)
    rng.integers(1, 21, size=(n_cons, n_vars)); rng.integers(100, 501, size=n_cons); rng.integers(1, 51, size=n_vars)
    extra = rng.integers(1, 51, size=(n_objectives - 1, n_vars)).astype(np.float64)
    m = dense_packing_lp_model(n_vars, n_cons, seed)
    m["name"] = f"DensePacking{n_objectives}obj_{n_vars}x{n_cons}_seed{seed}"
    m["optimize"] = {"profit": "max", **{f"attr{k}": "max" for k in range(1, n_objectives)}}
    for j, v in enumerate(m["variables"].values()):
        for k in range(1, n_objectives):
            v[f"attr{k}"] = float(extra[k - 1, j])
    return m


def mixed_lp_model(n_vars: int, n_cons: int, seed: int = 7, density: float = 0.7, frac_min: float = 0.3) -> dict:
    """generateRandomLP-like instance (problem-generator.ts:54-108) with a share of `min` rows so
    that phase 1 has work; rhs of `min` rows is kept small so most instances stay feasible."""
    rng = np.random.default_rng(seed)
    constraints, variables = {}, {f"x{j}": {"objective": float(rng.integers(1, 101))} for j in range(n_vars)}
    for i in range(n_cons):
        is_min = rng.random() < frac_min
        for j in range(n_vars):
            if rng.random() < density:
                variables[f"x{j}"][f"c{i}"] = float(rng.integers(1, 101))
        constraints[f"c{i}"] = {"min": float(rng.integers(10, 200))} if is_min else {"max": float(rng.integers(2000, 20000))}
    return {"name": f"MixedLP_{n_vars}x{n_cons}_seed{seed}", "optimize": "objective",
            "opType": "max" if rng.random() < 0.5 else "min", "constraints": constraints, "variables": variables}


def planted_infeasible_model(n_vars: int, n_cons: int, k: int, seed: int = 12345) -> dict:
    """An infeasible LP whose only irreducible infeasible subset is known: k - 1 rows `x_j <= 1` and one row
    `sum x_j >= k` over the same k - 1 variables (names `conflict*`), spread through the row order, plus a background
    of n_cons - k random packing rows (`max`, entries U{1..20} at density 0.5) on the other n_vars - k + 1 variables,
    each satisfied with a margin U{1..20} at an interior point x0 ~ U[0.5, 1.5].  The background is feasible and
    shares no variable with the planted rows, so it is in no infeasible subset."""
    assert 2 <= k <= n_cons and k - 1 < n_vars
    rng = np.random.default_rng(seed)
    n_bg = n_vars - (k - 1)
    planted_vars = [f"p{j}" for j in range(k - 1)]
    bg_vars = [f"x{j}" for j in range(n_bg)]
    planted_pos = set(int(i) for i in rng.choice(n_cons, size=k, replace=False))
    x0 = rng.uniform(0.5, 1.5, size=n_bg)
    variables = {v: {"objective": float(rng.integers(1, 51))} for v in planted_vars + bg_vars}
    constraints = {}
    p = 0
    for i in range(n_cons):
        if i in planted_pos:
            name = f"conflict{p}"
            if p < k - 1:
                constraints[name] = {"max": 1.0}
                variables[planted_vars[p]][name] = 1.0
            else:
                constraints[name] = {"min": float(k)}
                for v in planted_vars:
                    variables[v][name] = 1.0
            p += 1
            continue
        name = f"c{i}"
        a = np.where(rng.random(n_bg) < 0.5, rng.integers(1, 21, size=n_bg), 0).astype(np.float64)
        constraints[name] = {"max": float(np.ceil(a @ x0)) + float(rng.integers(1, 21))}
        for j in np.nonzero(a)[0]:
            variables[bg_vars[j]][name] = float(a[j])
    return {"name": f"Planted_{n_vars}x{n_cons}_k{k}_seed{seed}", "optimize": "objective", "opType": "max",
            "constraints": constraints, "variables": variables}


def infeasible_packing_arrays(n_vars: int, n_cons: int, n_demand: int, seed: int = 12345):
    """(A, b, c, lower) of infeasible_packing_model: n_cons rows in all, of which n_demand (lower[i] True) are demand
    rows at seeded positions in the row order and the others packing rows."""
    assert 0 <= n_demand <= n_cons and n_vars >= 1
    rng = np.random.default_rng(seed)
    A = rng.integers(1, 21, size=(n_cons, n_vars)).astype(np.float64)
    b = rng.integers(100, 501, size=n_cons).astype(np.float64)
    c = rng.integers(1, 51, size=n_vars).astype(np.float64)
    lower = np.zeros(n_cons, dtype=bool)
    lower[rng.choice(n_cons, size=n_demand, replace=False)] = True
    if n_demand < n_cons:
        cap = float(b[~lower].min())
        A[lower] = rng.integers(2, 5, size=(n_demand, n_vars)) / 4.0  # entries in {0.5, 0.75, 1}
        b[lower] = cap + rng.integers(1, 21, size=n_demand)
    return A, b, c, lower


def infeasible_packing_model(n_vars: int, n_cons: int, n_demand: int, seed: int = 12345) -> dict:
    """max c.x over a dense packing LP whose n_demand demand rows (`min`) make it infeasible by construction.  Packing
    rows are a_i.x <= b_i with a_ij ~ U{1..20} and b_i ~ U{100..500}; a demand row is d.x >= cap + U{1..20} with d_j in
    {0.5, 0.75, 1} and cap the smallest packing right-hand side.  Why no x >= 0 meets a demand row: every packing entry
    is >= 1, so sum_j x_j <= a_i.x <= b_i for every packing row, hence sum_j x_j <= cap; every d_j <= 1, so d.x <=
    sum_j x_j <= cap < the demand.  Each demand row starts below 0 in the tableau (it is stored negated), so they are
    the rows a repair crashes.  n_cons counts all rows; with n_demand == n_cons there is no packing row and the model
    is feasible."""
    A, b, c, lower = infeasible_packing_arrays(n_vars, n_cons, n_demand, seed)
    return dict(lp_model(A, b, c, lower), name=f"InfeasiblePacking_{n_vars}x{n_cons}_{n_demand}_seed{seed}")


def planted_unbounded_model(n_vars: int, n_cons: int, n_solo: int, n_pairs: int, seed: int = 12345) -> dict:
    """max c.x over a dense packing LP with planted leaks, unbounded by construction.  n_vars and n_cons count every
    variable and row.  The packing part has n_vars - n_solo - 2 n_pairs variables `x{j}` and n_cons - 2 n_pairs rows
    a_i.x <= b_i with a_ij ~ U{1..20}, b_i ~ U{100..500}: every entry is positive, so it is bounded on its own.  A solo
    leak `solo{k}` has no entry in any row.  A pair leak is `pairU{k}` and `pairV{k}` with the rows `u - v <= b1` and
    `v - u <= b2` (b ~ U{1..10}): either variable alone is blocked by the other's cap, and u + v runs away.  Every cost
    is U{1..50}.  The leak columns sit at seeded positions among the packing columns, u before v.  The irreducible set
    the one-at-a-time deletion filter over the columns returns is every solo leak plus the v of each pair: a cap on v
    alone bounds the pair, so the filter drops u first."""
    rng = np.random.default_rng(seed)
    n_pack, r_pack = n_vars - n_solo - 2 * n_pairs, n_cons - 2 * n_pairs
    if n_pack < 0 or r_pack < 0 or (n_pack > 0 and r_pack == 0):
        raise ValueError("planted_unbounded_model: more leaks than variables or rows, or no packing row")
    kinds = ["x"] * n_pack + ["solo"] * n_solo + ["pair"] * n_pairs
    order = rng.permutation(len(kinds))
    A = rng.integers(1, 21, size=(r_pack, n_pack)).astype(np.float64)
    b = rng.integers(100, 501, size=r_pack).astype(np.float64)
    constraints = {f"resource{i}": {"max": float(b[i])} for i in range(r_pack)}
    variables = {}
    j = k_solo = k_pair = 0
    for pos in order:
        kind = kinds[pos]
        if kind == "x":
            v = {"profit": float(rng.integers(1, 51))}
            for i in range(r_pack):
                v[f"resource{i}"] = float(A[i, j])
            variables[f"x{j}"] = v
            j += 1
        elif kind == "solo":
            variables[f"solo{k_solo}"] = {"profit": float(rng.integers(1, 51))}
            k_solo += 1
        else:
            k = k_pair
            b1, b2 = rng.integers(1, 11, size=2)
            constraints[f"pairA{k}"] = {"max": float(b1)}
            constraints[f"pairB{k}"] = {"max": float(b2)}
            variables[f"pairU{k}"] = {"profit": float(rng.integers(1, 51)), f"pairA{k}": 1.0, f"pairB{k}": -1.0}
            variables[f"pairV{k}"] = {"profit": float(rng.integers(1, 51)), f"pairA{k}": -1.0, f"pairB{k}": 1.0}
            k_pair += 1
    return {"name": f"PlantedUnbounded_{n_vars}x{n_cons}_{n_solo}_{n_pairs}_seed{seed}", "optimize": "profit",
            "opType": "max", "constraints": constraints, "variables": variables}


def planted_integer_conflict_model(n_vars: int, n_cons: int, k: int, seed: int = 12345) -> dict:
    """max c.x over a dense packing MIP with one planted parity equality, without an integer plan by construction.
    n_vars counts every variable `x{j}` (all integer), n_cons every row; the equality `parity` is two of them (its
    `min` row, then its `max` row) at a seeded position among the packing rows.  Packing rows are a_i.x <= b_i with
    a_ij ~ U{1..20} and b_i ~ U{100..500}; costs are U{1..50}.  The parity row is sum_j 2 x_j = 2m + 1, m ~ U{0..1},
    over k planted columns at seeded positions: an even sum is never odd, so no integer plan exists.  Dropping the
    `max` half leaves x_j = m + 1 at one planted column, dropping the `min` half leaves x = 0, and dropping the
    integrality of one planted column leaves x_j = m + 1/2 there; each satisfies every packing row (20 * 2 <= 100).
    So the only conflict is both parity rows plus the integrality of the k planted columns."""
    rng = np.random.default_rng(seed)
    r_pack = n_cons - 2
    if k < 1 or k > n_vars or r_pack < 0:
        raise ValueError("planted_integer_conflict_model: needs 1 <= k <= n_vars and n_cons >= 2")
    m = int(rng.integers(0, 2))
    planted = set(int(j) for j in rng.choice(n_vars, size=k, replace=False))
    at = int(rng.integers(0, r_pack + 1))
    A = rng.integers(1, 21, size=(r_pack, n_vars)).astype(np.float64)
    b = rng.integers(100, 501, size=r_pack).astype(np.float64)
    constraints = {}
    for i in range(r_pack + 1):
        if i == at:
            constraints["parity"] = {"equal": float(2 * m + 1)}
        if i < r_pack:
            constraints[f"resource{i}"] = {"max": float(b[i])}
    variables = {}
    for j in range(n_vars):
        v = {"profit": float(rng.integers(1, 51))}
        for i in range(r_pack):
            v[f"resource{i}"] = float(A[i, j])
        if j in planted:
            v["parity"] = 2.0
        variables[f"x{j}"] = v
    return {"name": f"PlantedIntegerConflict_{n_vars}x{n_cons}_{k}_seed{seed}", "optimize": "profit", "opType": "max",
            "constraints": constraints, "variables": variables, "ints": {f"x{j}": 1 for j in range(n_vars)}}


def knapsack_mip_model(n_items: int, n_cons: int, seed: int = 12345, tolerance: float = 0.0) -> dict:
    """Multi-dimensional 0/1 knapsack (SURVEY.md 8d config 5): a_ij ~ U{1..50} dense,
    b_i = floor(0.5 * sum_j a_ij), c_j ~ U{1..50}; every binary adds an `x <= 1` row
    (model.ts:392-395), so the root tableau is (n_cons + n_items + 1) x (n_items + 1)."""
    rng = np.random.default_rng(seed)
    A = rng.integers(1, 51, size=(n_cons, n_items))
    c = rng.integers(1, 51, size=n_items)
    constraints = {f"k{i}": {"max": float(np.floor(0.5 * A[i].sum()))} for i in range(n_cons)}
    variables, binaries = {}, {}
    for j in range(n_items):
        v = {"value": float(c[j])}
        for i in range(n_cons):
            v[f"k{i}"] = float(A[i, j])
        variables[f"item{j}"] = v
        binaries[f"item{j}"] = 1
    m = {"name": f"Knapsack_{n_items}x{n_cons}_seed{seed}", "optimize": "value", "opType": "max",
         "constraints": constraints, "variables": variables, "binaries": binaries}
    if tolerance:
        m["tolerance"] = tolerance
    return m


def half_tie_mip_model(n_ints: int, group: int = 8, seed: int = 12345) -> dict:
    """A MIP whose LP relaxation keeps many basic integer variables at exactly k + 1/2: integer x_i with a row
    2 x_i <= 2 u_i + 1 (u_i ~ U{0..3}) and cost c_i ~ U{1..9} (max), coupled by packing rows over consecutive groups of
    `group` variables.  Every other packing row allows sum (u_i + 1/2) over its group; the others allow 1/2 less, so
    one variable of the group stays integral.  Whichever variable branch-and-cut branches on, the other fractions
    stay 1/2, and the choice is decided by the position tie-break of getMostFractionalVar at nearly every node.
    Root tableau: (n_ints + ceil(n_ints / group) + 1) x (n_ints + 1)."""
    rng = np.random.default_rng(seed)
    u = rng.integers(0, 4, size=n_ints)
    c = rng.integers(1, 10, size=n_ints)
    variables = {f"x{i}": {"value": float(c[i]), f"half{i}": 2.0} for i in range(n_ints)}
    constraints = {f"half{i}": {"max": float(2 * u[i] + 1)} for i in range(n_ints)}
    for g, g0 in enumerate(range(0, n_ints, group)):
        members = range(g0, min(n_ints, g0 + group))
        cap = float(sum(u[i] for i in members)) + 0.5 * len(members) - (0.5 if g % 2 else 0.0)
        constraints[f"pack{g}"] = {"max": cap}
        for i in members:
            variables[f"x{i}"][f"pack{g}"] = 1.0
    return {"name": f"HalfTieMIP_{n_ints}_seed{seed}", "optimize": "value", "opType": "max",
            "constraints": constraints, "variables": variables, "ints": {f"x{i}": 1 for i in range(n_ints)}}


def priority_tie_mip_model(n_objectives: int, n_items: int = 10, seed: int = 2) -> dict:
    """A 0/1 MIP whose integral optima tie on the main objective and are told apart only by soft constraints: maximise
    the number of items picked under one capacity row (weights U{2..5}, capacity half their sum plus one), so every
    optimal plan picks the same number of items.  Soft constraint p = 1..n_objectives (`max: 0`, priority p, weight
    U{1..3}) penalises picked items: priorities 1..n_objectives - 1 cover every item, so every optimal plan violates
    them alike, and the last covers a random third of the items and decides between the optima.  Each distinct priority
    is one optional objective (Tableau.optionalObjectives), so the model has exactly n_objectives of them, and the
    branch-and-cut incumbent among tied plans is chosen by comparing them (branch-and-cut.ts:107-127)."""
    rng = np.random.default_rng(seed)
    w = rng.integers(2, 6, size=n_items)
    variables = {f"x{j}": {"count": 1.0, "cap": float(w[j])} for j in range(n_items)}
    constraints = {"cap": {"max": float(w.sum() // 2 + 1)}}
    for p in range(1, n_objectives + 1):
        items = range(n_items) if p < n_objectives else rng.choice(n_items, size=max(1, n_items // 3), replace=False)
        for j in items:
            variables[f"x{j}"][f"soft{p}"] = 1.0
        constraints[f"soft{p}"] = {"max": 0.0, "priority": p, "weight": float(rng.integers(1, 4))}
    return {"name": f"PriorityTieMIP_{n_objectives}_{n_items}_seed{seed}", "optimize": "count", "opType": "max",
            "constraints": constraints, "variables": variables, "binaries": {f"x{j}": 1 for j in range(n_items)}}


# ---- the reference's stress families (solver.stress.test.ts:41-215 solves them at 10..50 variables) ----------
# Same shapes and distributions as problem-generator.ts's families, drawn from numpy's stream; every model is a
# plain jsLPSolver JSON dict, so every implementation that is compared (and an outside solver) sees the same instance.

def _sparse_columns(rng, names, rows, density, lo, hi):
    """variables[name][row] = U{lo..hi} wherever a Bernoulli(density) mask is set."""
    mask = rng.random((len(names), len(rows))) < density
    coef = rng.integers(lo, hi + 1, size=mask.shape)
    return [{rows[i]: float(coef[j, i]) for i in np.nonzero(mask[j])[0]} for j in range(len(names))]


def random_lp_model(n_vars: int, n_cons: int, seed: int = 12345, density: float = 0.6) -> dict:
    """generateRandomLP (problem-generator.ts:54-108): objective and entries U{1..100}, right-hand sides U{10..1000},
    each row `max` or `min` with equal odds, sense max or min with equal odds.  Often infeasible or unbounded: the
    reference's test only asks the solver to finish with a verdict."""
    rng = np.random.default_rng(seed)
    names, rows = [f"x{j}" for j in range(n_vars)], [f"c{i}" for i in range(n_cons)]
    cols = _sparse_columns(rng, names, rows, density, 1, 100)
    obj = rng.integers(1, 101, size=n_vars)
    rhs, side = rng.integers(10, 1001, size=n_cons), rng.random(n_cons) < 0.5
    return {"name": f"RandomLP_{n_vars}x{n_cons}_seed{seed}", "optimize": "objective",
            "opType": "max" if rng.random() < 0.5 else "min",
            "constraints": {rows[i]: {"max" if side[i] else "min": float(rhs[i])} for i in range(n_cons)},
            "variables": {names[j]: {"objective": float(obj[j]), **cols[j]} for j in range(n_vars)}}


def random_mip_model(n_vars: int, n_cons: int, seed: int = 12345, density: float = 0.5, integer_fraction: float = 0.3) -> dict:
    """generateRandomMIP (problem-generator.ts:113-145): the random LP with a Bernoulli(integer_fraction) share of
    its variables declared `ints`."""
    m = random_lp_model(n_vars, n_cons, seed, density)
    pick = np.random.default_rng(seed + 1).random(n_vars) < integer_fraction
    m["name"] = m["name"].replace("RandomLP", "RandomMIP")
    if pick.any():
        m["ints"] = {f"x{j}": 1 for j in np.nonzero(pick)[0]}
    return m


def single_knapsack_model(n_items: int, seed: int = 12345) -> dict:
    """generateKnapsack (problem-generator.ts:147-186): value, weight ~ U{1..50}, one capacity row U{100..500}."""
    rng = np.random.default_rng(seed)
    vw = rng.integers(1, 51, size=(n_items, 2))
    return {"name": f"Knapsack_{n_items}_seed{seed}", "optimize": "value", "opType": "max",
            "constraints": {"capacity": {"max": float(rng.integers(100, 501))}},
            "variables": {f"item{j}": {"value": float(vw[j, 0]), "weight": float(vw[j, 1])} for j in range(n_items)},
            "binaries": {f"item{j}": 1 for j in range(n_items)}}


def set_cover_model(n_sets: int, n_elements: int, seed: int = 12345, density: float = 0.4) -> dict:
    """generateSetCover (problem-generator.ts:188-236): binary sets with cost U{1..20}, every element covered at
    least once (`min: 1` rows, so phase 1 runs at the root and after most branches); may be infeasible."""
    rng = np.random.default_rng(seed)
    cost = rng.integers(1, 21, size=n_sets)
    member = rng.random((n_sets, n_elements)) < density
    return {"name": f"SetCover_{n_sets}x{n_elements}_seed{seed}", "optimize": "cost", "opType": "min",
            "constraints": {f"element{e}": {"min": 1.0} for e in range(n_elements)},
            "variables": {f"set{s}": {"cost": float(cost[s]), **{f"element{e}": 1.0 for e in np.nonzero(member[s])[0]}}
                          for s in range(n_sets)},
            "binaries": {f"set{s}": 1 for s in range(n_sets)}}


def transportation_model(n_sources: int, n_destinations: int, seed: int = 12345) -> dict:
    """generateTransportation (problem-generator.ts:238-295): supplies U{50..200} as `max` rows, equal demands
    floor(total / destinations) as `min` rows, unit costs U{1..100}; always feasible."""
    rng = np.random.default_rng(seed)
    supply = rng.integers(50, 201, size=n_sources)
    cost = rng.integers(1, 101, size=(n_sources, n_destinations))
    demand = float(int(supply.sum()) // n_destinations)
    constraints = {f"supply{s}": {"max": float(supply[s])} for s in range(n_sources)}
    constraints.update({f"demand{d}": {"min": demand} for d in range(n_destinations)})
    return {"name": f"Transportation_{n_sources}x{n_destinations}_seed{seed}", "optimize": "cost", "opType": "min",
            "constraints": constraints,
            "variables": {f"ship_{s}_to_{d}": {"cost": float(cost[s, d]), f"supply{s}": 1.0, f"demand{d}": 1.0}
                          for s in range(n_sources) for d in range(n_destinations)}}


def resource_allocation_model(n_activities: int, n_resources: int, seed: int = 12345, density: float = 0.6) -> dict:
    """generateResourceAllocation (problem-generator.ts:297-340): profit U{1..50}, usage U{1..20} at the given
    density, capacities U{100..500}; the sparse cousin of dense_packing_lp_model."""
    rng = np.random.default_rng(seed)
    names, rows = [f"activity{a}" for a in range(n_activities)], [f"resource{r}" for r in range(n_resources)]
    profit = rng.integers(1, 51, size=n_activities)
    cols = _sparse_columns(rng, names, rows, density, 1, 20)
    cap = rng.integers(100, 501, size=n_resources)
    return {"name": f"ResourceAllocation_{n_activities}x{n_resources}_seed{seed}", "optimize": "profit", "opType": "max",
            "constraints": {rows[r]: {"max": float(cap[r])} for r in range(n_resources)},
            "variables": {names[a]: {"profit": float(profit[a]), **cols[a]} for a in range(n_activities)}}


def stress_suite(seed: int = 12345):
    """The instances of solver.stress.test.ts:41-132 (sizes and options as there), as (label, model) pairs."""
    import math
    out = []
    for n, m in ((15, 8), (30, 15), (50, 25)):
        out.append((f"random_lp_{n}x{m}", random_lp_model(n, m, seed, 0.6)))
        out.append((f"resource_allocation_{n}x{m}", resource_allocation_model(n, m, seed)))
        k = math.ceil(math.sqrt(n))
        out.append((f"transportation_{k}x{k}", transportation_model(k, k, seed)))
    for n, m in ((10, 5), (20, 10), (30, 15)):
        out.append((f"random_mip_{n}x{m}", random_mip_model(n, m, seed, 0.5, 0.3)))
        out.append((f"knapsack_{n}", single_knapsack_model(n, seed)))
    for n, m in ((10, 6), (15, 10), (20, 12)):
        out.append((f"set_cover_{n}x{m}", set_cover_model(n, m, seed, 0.4)))
    return out

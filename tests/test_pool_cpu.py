"""The solution pool (DESIGN.md section 2m) without a GPU: the sequential search of tests/pool_oracle.py against brute
force (every integer assignment of small models, its continuous completion solved by SciPy's HiGHS), Sudoku4x4's
completions against a backtracking solver, Pool()'s refusals and argument checks, and the jslp_pool_batch / jslp_fix
declarations against the ctypes mirrors."""
from __future__ import annotations

import gzip
import itertools
import json
import os
import re
import subprocess

import numpy as np
import pytest

import pool_oracle as O
from jslpsolver_b200 import problems

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _oracle_lib():
    from oracle import ref_model
    ref_model.build_oracle()


def fixture(name: str) -> dict:
    bundle = json.load(gzip.open(os.path.join(ROOT, "tests", "golden", "sanity_fixtures.json.gz")))
    for f in bundle["fixtures"] + bundle["readme"]:
        if f["file"] == name:
            return f["model"]
    raise KeyError(name)


# ---- brute force ------------------------------------------------------------------------------------------------
def arrays(jm: dict):
    """(names, integer names, c (minimised), A_ub, b_ub, upper bounds) of a single-objective JSON model."""
    names = list(jm["variables"])
    ints = [v for v in names if jm.get("ints", {}).get(v) or jm.get("binaries", {}).get(v)]
    sign = -1.0 if jm.get("opType") == "max" else 1.0
    c = np.array([sign * float(jm["variables"][v].get(jm["optimize"], 0.0)) for v in names])
    A, b = [], []
    for cname, spec in jm["constraints"].items():
        row = np.array([float(jm["variables"][v].get(cname, 0.0)) for v in names])
        lo, hi = (spec["equal"], spec["equal"]) if "equal" in spec else (spec.get("min"), spec.get("max"))
        if hi is not None:
            A.append(row); b.append(float(hi))
        if lo is not None:
            A.append(-row); b.append(-float(lo))
    upper = [1.0 if jm.get("binaries", {}).get(v) else None for v in names]
    return names, ints, c, np.array(A), np.array(b), upper


def completion(jm: dict, z: dict):
    """f(z) (minimisation sense) of the integer assignment z, or None when its continuous LP is infeasible."""
    from scipy.optimize import linprog
    names, _, c, A, b, upper = arrays(jm)
    bounds = [(z[v], z[v]) if v in z else (0.0, upper[i]) for i, v in enumerate(names)]
    res = linprog(c, A_ub=A, b_ub=b, bounds=bounds, method="highs")
    return res.fun if res.status == 0 else None


def box(jm: dict) -> dict:
    """The integer range of every integer variable: 0 .. floor(its LP maximum)."""
    from scipy.optimize import linprog
    names, ints, _, A, b, upper = arrays(jm)
    out = {}
    for v in ints:
        e = np.zeros(len(names))
        e[names.index(v)] = -1.0
        res = linprog(e, A_ub=A, b_ub=b, bounds=[(0.0, u) for u in upper], method="highs")
        out[v] = None if res.status != 0 else int(np.floor(-res.fun + 1e-7))
    return out


def enumerate_all(jm: dict) -> list:
    """[(f, z)] over every feasible integer assignment, best first."""
    rng = box(jm)
    if any(r is None for r in rng.values()):  # infeasible relaxation
        return []
    ints = list(rng)
    out = []
    for vals in itertools.product(*[range(rng[v] + 1) for v in ints]):
        z = dict(zip(ints, vals))
        f = completion(jm, z)
        if f is not None:
            out.append((f, z))
    out.sort(key=lambda e: e[0])
    return out


def enumerable_random_mips(n: int, limit: int = 400) -> list:
    """The first n seeded random MIPs (4 variables, 3 rows) whose integer box has at most `limit` points and whose
    relaxation is bounded and feasible."""
    from scipy.optimize import linprog
    found = []
    for seed in range(1000):
        jm = problems.random_mip_model(4, 3, seed=seed, integer_fraction=0.6)
        if not jm.get("ints"):
            continue
        names, _, c, A, b, upper = arrays(jm)
        if linprog(c, A_ub=A, b_ub=b, bounds=[(0, u) for u in upper], method="highs").status != 0:
            continue
        rng = box(jm)
        if any(r is None for r in rng.values()) or np.prod([r + 1 for r in rng.values()]) > limit:
            continue
        found.append(jm)
        if len(found) == n:
            break
    return found


def models() -> list:
    return (enumerable_random_mips(4) + [problems.single_knapsack_model(7, seed=s) for s in (1, 2)] +
            [problems.set_cover_model(7, 5, seed=s) for s in (3, 4)] + [problems.half_tie_mip_model(5, group=3)])


def same_as_brute_force(pool: dict, brute: list, rel=1e-7):
    """Pool values are the k smallest f in order, and each tie class the pool covers whole is the same set."""
    sols = pool["solutions"]
    assert len(sols) <= len(brute)
    scale = max([1.0] + [abs(f) for f, _ in brute])
    for s, (f, _) in zip(sols, brute):
        assert abs(s["evaluation"] - f) <= rel * scale, (s["evaluation"], f)
    key = lambda z: tuple(sorted(z.items()))
    got = [key({v: s["values"][v] for v in brute[0][1]}) for s in sols] if sols else []
    assert len(set(got)) == len(got), "the pool lists an assignment twice"
    i = 0
    while i < len(sols):
        f0 = brute[i][0]
        cls = [key(z) for f, z in brute if abs(f - f0) <= rel * scale]
        mine = [g for g, s in zip(got, sols) if abs(s["evaluation"] - f0) <= rel * scale]
        if i + len(cls) <= len(sols):
            assert sorted(mine) == sorted(cls)
        else:
            assert set(mine) <= set(cls)
        i += len(mine)


@pytest.mark.parametrize("jm", models(), ids=lambda m: m["name"])
def test_oracle_pool_lists_the_k_best_assignments(jm):
    brute = enumerate_all(jm)
    for k in (1, 3, 8):
        got = O.pool(jm, k=k)
        same_as_brute_force(got, brute)
        assert got["stop"] == ("k" if len(brute) >= k else "exhausted") or \
            (got["stop"] == "gap" and len(got["solutions"]) < k), got["stop"]


@pytest.mark.parametrize("jm", models(), ids=lambda m: m["name"])
def test_oracle_pool_exhausted_lists_every_feasible_assignment(jm):
    brute = enumerate_all(jm)
    got = O.pool(jm, k=10 ** 6, absolute_gap=1e12)
    assert got["stop"] == "exhausted"
    assert len(got["solutions"]) == len(brute)
    same_as_brute_force(got, brute)


@pytest.mark.parametrize("jm", models(), ids=lambda m: m["name"])
def test_oracle_pool_stops_at_the_allowance(jm):
    brute = enumerate_all(jm)
    fs = sorted({round(f, 6) for f, _ in brute})
    if len(fs) < 3:
        pytest.skip("fewer than three distinct values")
    fstar = brute[0][0]
    for cut in (fs[1], fs[2]):  # an allowance halfway between two consecutive values
        nxt = fs[fs.index(cut) + 1] if fs.index(cut) + 1 < len(fs) else cut + 2
        t = (cut + nxt) / 2 - fstar
        want = sum(1 for f, _ in brute if f <= fstar + t)
        got = O.pool(jm, k=10 ** 6, absolute_gap=t)
        assert len(got["solutions"]) == want
        assert got["stop"] == ("gap" if want < len(brute) else "exhausted")
        if fstar != 0:
            g = O.pool(jm, k=10 ** 6, gap=t / abs(fstar))
            assert len(g["solutions"]) == want and g["allowance"] == pytest.approx(t)
    exact = O.pool(jm, k=10 ** 6)  # allowance 0: every optimal plan
    assert len(exact["solutions"]) == sum(1 for f, _ in brute if abs(f - fstar) <= 1e-7 * max(1, abs(fstar)))


def test_oracle_pool_limit_is_a_prefix():
    jm = problems.single_knapsack_model(8, seed=5)
    full = O.pool(jm, k=10 ** 6, absolute_gap=1e12)
    for cap in (1, 5, 17):
        part = O.pool(jm, k=10 ** 6, absolute_gap=1e12, max_nodes=cap)
        assert part["stop"] == "limit" and part["nodes"] >= cap
        assert [s["z"] for s in part["solutions"]] == [s["z"] for s in full["solutions"]][:len(part["solutions"])]


def sudoku_completions(jm: dict) -> list:
    """Every completion of the 4x4 Sudoku model by backtracking over its own rows: binaries x_rcv, every constraint
    an `equal: 1` over the binaries it names."""
    names = list(jm["variables"])
    rows = [[v for v in names if jm["variables"][v].get(c)] for c, spec in jm["constraints"].items()]
    for c, spec in jm["constraints"].items():
        assert spec == {"equal": 1}, (c, spec)
    out, chosen = [], set()

    def go(pending):
        if not pending:
            out.append(frozenset(chosen))
            return
        row = min(pending, key=lambda r: len(r))  # the row with the fewest candidates
        for v in row:
            hit = [r for r in pending if v in r]
            rest = [[u for u in r if not any(u in h for h in hit)] for r in pending if v not in r]
            if any(not r for r in rest):
                continue
            chosen.add(v)
            go(rest)
            chosen.discard(v)

    go(rows)
    return out


def test_oracle_pool_lists_every_sudoku_completion():
    jm = fixture("Sudoku4x4.json")
    want = sudoku_completions(jm)
    assert len(want) >= 1
    got = O.pool(jm, k=1000)
    assert got["stop"] == "exhausted"
    sets = [frozenset(v for v, x in s["values"].items() if x == 1.0) for s in got["solutions"]]
    assert len(set(sets)) == len(sets) and set(sets) == set(want)


# ---- front end ----------------------------------------------------------------------------------------------------
KNAP = {"optimize": "v", "opType": "max", "constraints": {"w": {"max": 5}},
        "variables": {"a": {"v": 3, "w": 2}, "b": {"v": 4, "w": 3}}, "ints": {"a": 1, "b": 1}}


@pytest.mark.parametrize("model, kw, match", [
    ({**KNAP, "ints": {}}, {}, "integer or binary"),
    ({**KNAP, "constraints": {"w": {"max": 5, "weight": 2}}}, {}, "soft constraints"),
    ({**KNAP, "optimize": {"v": "max", "w": "min"}}, {}, "one objective"),
    ({**KNAP, "unrestricted": {"a": 1}}, {}, "unrestricted"),
    (KNAP, {"k": 0}, "k= must be >= 1"),
    (KNAP, {"k": 2.5}, "k= takes an integer"),
    (KNAP, {"k": True}, "k= takes an integer"),
    (KNAP, {"gap": -0.1}, "gap= must be finite and >= 0"),
    (KNAP, {"absolute_gap": float("nan")}, "absolute_gap= must be finite"),
    (KNAP, {"max_nodes": 0}, "max_nodes= must be >= 1"),
    (KNAP, {"width": 0}, "width= must be >= 1"),
    ([], {}, "requires a model"),
    ("model", {}, "takes a JSON model"),
])
def test_pool_refusals(model, kw, match):
    import jslpsolver_b200 as J
    with pytest.raises(ValueError, match=match):
        J.Pool(model, **kw)


def test_pool_region_rules_match_the_restatement():
    """pool.Search builds the same children, in the same order, as the literal restatement."""
    from jslpsolver_b200.pool import Region, Search
    jm = problems.half_tie_mip_model(6, group=3)
    p = O.Problem(jm)
    s = Search(p.ints, p.col_of, p.binaries)
    rng = np.random.default_rng(3)
    for _ in range(50):
        labs = list(p.ints)
        rng.shuffle(labs)
        fixed = labs[:2]
        fixings = [(p.col_of[l], float(rng.integers(0, 3))) for l in fixed]
        cuts = [(int(rng.integers(0, 2)), int(l), float(rng.integers(0, 4))) for l in labs[2:] if rng.random() < 0.5]
        r = Region(fixings, cuts)
        if rng.random() < 0.5:
            r.integral, r.branch_var, r.branch_value = False, int(labs[3]), float(rng.integers(0, 5)) + 0.5
            res = {"is_integral": False, "branch_var": r.branch_var, "branch_value": r.branch_value}
        else:
            H = 1 + len(labs) - 2
            r.integral = True
            r.vrow = np.array([-1] + labs[2:], dtype=np.int32)[:H]
            r.rhs = np.array([0.0] + [float(rng.integers(0, 4)) for _ in labs[2:]])[:H]
            res = {"is_integral": True, "vrow": r.vrow, "rhs": r.rhs}
        assert s.children(r) == O.children(p, fixings, cuts, res)


# ---- C ABI --------------------------------------------------------------------------------------------------------
def _types(name):
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", header)
    assert proto, f"{name} is not declared"
    params = [p.strip() for p in proto.group(1).split(",")]
    return [re.sub(r"\s+", " ", p.rsplit("*", 1)[0]).strip() + " *" if "*" in p else p.rsplit(" ", 1)[0]
            for p in params]


def test_pool_batch_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    C, P = _lib.C, _lib.C.c_void_p
    want = ["jslp_tab *", "const jslp_fix *", "const int32_t *", "const jslp_cut *", "const int32_t *", "int", "int",
            "int", "int32_t *", "double *", "int32_t *", "int32_t *", "double *", "int32_t *", "double *", "int32_t *"]
    assert _types("jslp_pool_batch") == want
    (_, res, got), = [s for s in _lib.SYMBOLS if s[0] == "jslp_pool_batch"]
    assert res is C.c_int and got == [P] * 5 + [C.c_int] * 3 + [P] * 8


def test_fix_struct_matches_the_header(tmp_path):
    import ctypes as C
    from jslpsolver_b200 import _lib
    src = tmp_path / "fix.c"
    src.write_text("\n".join([
        "#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "jslp_b200.h")}"',
        "int main(void) {",
        'printf("%zu %zu %zu\\n", sizeof(jslp_fix), offsetof(jslp_fix, column), offsetof(jslp_fix, value));',
        "return 0; }"]))
    exe = tmp_path / "fix"
    subprocess.run(["gcc", "-std=c11", "-o", str(exe), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [C.sizeof(_lib.Fix), _lib.Fix.column.offset, _lib.Fix.value.offset]

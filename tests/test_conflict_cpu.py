"""The MIP conflict (DESIGN.md section 2n) without a GPU: the sequential restatement of tests/conflict_oracle.py against
SciPy's HiGHS (the conflict has no integer plan, dropping any member gives one, every witness breaks only its own
member), planted conflicts recovered exactly, the host search of jslpsolver_b200/conflict.py driven by the oracle at
several widths and depths against the restatement, the max_nodes limit, Conflict()'s refusals, and the
jslp_conflict_batch declaration against the ctypes mirror."""
from __future__ import annotations

import functools
import gzip
import itertools
import json
import os
import re

import numpy as np
import pytest

import conflict_oracle as O
from jslpsolver_b200 import conflict, problems

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _oracle_lib():
    from oracle import ref_model
    ref_model.build_oracle()


def fixture(name: str) -> dict:
    bundle = json.load(gzip.open(os.path.join(ROOT, "tests", "golden", "sanity_fixtures.json.gz")))
    for f in bundle["fixtures"] + bundle["readme"]:
        if f["file"] == name:
            return json.loads(json.dumps(f["model"]))
    raise KeyError(name)


# ---- models -------------------------------------------------------------------------------------------------------
EXAMPLE = {"optimize": "cost", "opType": "min",
           "constraints": {"pair": {"equal": 3}, "cap": {"max": 1}},
           "variables": {"x": {"pair": 2, "cost": 1}, "y": {"pair": 2, "cap": 1, "cost": 1}},
           "ints": {"x": 1, "y": 1}}


def exact_knapsack(weights, seed: int) -> dict:
    """Binary items that must fill a capacity exactly, at a capacity no subset of the weights reaches."""
    sums = {sum(s) for n in range(len(weights) + 1) for s in itertools.combinations(weights, n)}
    rng = np.random.default_rng(seed)
    cap = int(rng.choice([c for c in range(1, sum(weights)) if c not in sums]))
    return {"optimize": "value", "opType": "max", "constraints": {"fill": {"equal": cap}},
            "variables": {f"item{i}": {"fill": w, "value": int(rng.integers(1, 20))} for i, w in enumerate(weights)},
            "binaries": {f"item{i}": 1 for i in range(len(weights))}}


def berlin_with_parity() -> dict:
    jm = fixture("Integer Berlin Air Lift Problem.json")
    jm["constraints"]["parity"] = {"equal": 3}  # 2 brit = 3: the relaxation takes brit = 1.5
    jm["variables"]["brit"]["parity"] = 2
    return jm


def infeasible_berlin_with_ints() -> dict:
    jm = fixture("Infeasible Berlin Air Lift Problem.json")
    jm["ints"] = {"brit": 1, "yank": 1}
    return jm


def sudoku_with_contradictory_clue() -> dict:
    """Sudoku4x4 with two givens and a clue that puts half a digit into each of two cells: the clue's rows and the two
    cells' integrality conflict, while the LP relaxation keeps a plan."""
    jm = fixture("Sudoku4x4.json")
    for name, var in (("given11", "x111"), ("given23", "x234")):
        jm["constraints"][name] = {"equal": 1}
        jm["variables"][var][name] = 1
    jm["constraints"]["clue"] = {"equal": 1}
    jm["variables"]["x122"]["clue"] = 2
    jm["variables"]["x343"]["clue"] = 2
    return jm


@functools.lru_cache(maxsize=None)
def random_infeasible_mips(n: int) -> list:
    """The first n seeded small random MIPs (4 integer variables, 3 rows with integer coefficients) that HiGHS finds
    without an integer plan."""
    out = []
    for seed in range(500):
        rng = np.random.default_rng(seed)
        names = [f"v{j}" for j in range(4)]
        cons = {}
        for i in range(3):
            kind = ["equal", "max", "min"][int(rng.integers(0, 3))]
            cons[f"r{i}"] = {kind: int(rng.integers(1, 12))}
        variables = {v: {"obj": int(rng.integers(1, 9))} for v in names}
        for i in range(3):
            for v in names:
                if rng.random() < 0.7:
                    variables[v][f"r{i}"] = int(rng.integers(-3, 7))
        jm = {"optimize": "obj", "opType": "max", "constraints": cons, "variables": variables,
              "ints": {v: 1 for v in names}}
        p = O.Problem(jm)
        if not feasible(p, p.rows, p.ints) and len(out) < n:
            out.append(jm)
        if len(out) == n:
            return out
    raise AssertionError("too few infeasible random MIPs")


# ---- HiGHS --------------------------------------------------------------------------------------------------------
def feasible(p: O.Problem, rows, J) -> bool:
    """Whether the rows (of the initial tableau: M[r,1:] x <= M[r,0]) have a plan x >= 0 integral on the labels J."""
    from scipy.optimize import Bounds, LinearConstraint, milp
    W = p.M.shape[1]
    col = {int(p.vcol[c]): c - 1 for c in range(1, W)}
    integrality = np.zeros(W - 1)
    for j in J:
        integrality[col[j]] = 1
    rows = list(rows)
    cons = [LinearConstraint(p.M[rows, 1:], -np.inf, p.M[rows, 0])] if rows else []
    res = milp(np.zeros(W - 1), constraints=cons, integrality=integrality, bounds=Bounds(0, np.inf))
    assert res.status in (0, 2), res.message
    return res.status == 0


def point(p: O.Problem, w: dict) -> np.ndarray:
    W = p.M.shape[1]
    x = np.zeros(W - 1)
    col = {int(p.vcol[c]): c - 1 for c in range(1, W)}
    for r in range(1, len(w["vrow"])):
        if int(w["vrow"][r]) in col:
            x[col[int(w["vrow"][r])]] = w["rhs"][r]
    return x


def check_conflict(res: dict) -> None:
    """No integer plan; a plan once any member is dropped; every witness satisfies every other member and breaks its
    own, at the precision."""
    p, B, J = res["problem"], res["rows"], res["ints"]
    assert not feasible(p, B, J)
    for s in B:
        assert feasible(p, [r for r in B if r != s], J), f"row {s} is not needed"
    for j in J:
        assert feasible(p, B, [x for x in J if x != j]), f"the integrality of label {j} is not needed"
    W = p.M.shape[1]
    col = {int(p.vcol[c]): c - 1 for c in range(1, W)}
    tol = 1e-6

    def holds(x, r):
        return p.M[r, 1:] @ x <= p.M[r, 0] + tol * (1 + abs(p.M[r, 0]))

    def integral(x, j):
        return abs(x[col[j]] - round(x[col[j]])) <= tol

    for s, w in res["row_witness"].items():
        if w is None:
            continue
        x = point(p, w)
        assert (x >= -tol).all() and all(holds(x, r) for r in B if r != s) and all(integral(x, j) for j in J)
        assert not holds(x, s), f"the witness of row {s} does not break it"
    for j, w in res["int_witness"].items():
        if w is None:
            continue
        x = point(p, w)
        assert (x >= -tol).all() and all(holds(x, r) for r in B) and all(integral(x, i) for i in J if i != j)
        assert not integral(x, j), f"the witness of label {j} is integral there"


CASES = {
    "example": lambda: EXAMPLE,
    "berlin_parity": berlin_with_parity,
    "berlin_infeasible": infeasible_berlin_with_ints,
    "knapsack3": lambda: exact_knapsack([6, 10, 15], 1),
    "knapsack5": lambda: exact_knapsack([8, 12, 18, 22, 30], 2),
    "sudoku": sudoku_with_contradictory_clue,
    **{f"random{i}": (lambda i=i: json.loads(json.dumps(random_infeasible_mips(3)[i]))) for i in range(3)},
    **{f"planted{a}": (lambda a=a: problems.planted_integer_conflict_model(*a)) for a in
       [(6, 5, 2, 1), (12, 10, 3, 2), (30, 40, 4, 3)]},
}


@pytest.mark.parametrize("case", list(CASES))
def test_restatement_is_an_irreducible_conflict(case):
    res = O.conflict(CASES[case]())
    assert res["verdict"] == O.INFEASIBLE and res["irreducible"]
    check_conflict(res)


def test_the_example_is_the_documented_conflict():
    out = O.named(O.conflict(EXAMPLE))
    assert [(c["name"], c["type"], c["rhs"]) for c in out["constraints"]] == [("pair", "min", 3), ("pair", "max", 3)]
    assert out["bounds"] == [] and [i["variable"] for i in out["integers"]] == ["x", "y"]
    assert out["names"] == ["pair"] and out["relaxation"] == "feasible" and out["irreducible"]
    assert out["integers"][0]["witness"]["values"]["x"] == 1.5


def test_relaxation_infeasible_case_starts_from_the_certificate():
    out = O.named(O.conflict(infeasible_berlin_with_ints()))
    assert out["relaxation"] == "infeasible" and out["integers"] == []


def test_knapsack_conflict_names_the_binary_bounds():
    out = O.named(O.conflict(exact_knapsack([6, 10, 15], 1)))
    assert out["names"] == ["fill"] and all(b["type"] == "max" and b["rhs"] == 1 for b in out["bounds"])


@pytest.mark.parametrize("args", [(6, 5, 1, 1), (6, 5, 2, 1), (12, 10, 3, 2), (30, 40, 4, 3), (40, 60, 5, 4)])
def test_planted_conflict_is_exactly_the_planted_set(args):
    jm = problems.planted_integer_conflict_model(*args)
    out = O.named(O.conflict(jm))
    planted = sorted(v for v, coefs in jm["variables"].items() if "parity" in coefs)
    assert [(c["name"], c["type"]) for c in out["constraints"]] == [("parity", "min"), ("parity", "max")]
    assert out["bounds"] == [] and sorted(i["variable"] for i in out["integers"]) == planted
    assert out["relaxation"] == "feasible" and out["irreducible"]


# ---- the host search against the restatement ------------------------------------------------------------------------
def oracle_evaluate(p: O.Problem, log: list):
    def evaluate(specs):
        log.append(len(specs))
        out = []
        for rows, J, cuts in specs:
            r = O.node(p, rows, J, cuts)
            cycled = r["status"] == conflict.NODE_CYCLED
            out.append(conflict.Node(r["status"], r["is_integral"], r["branch_var"], r["branch_value"], r["pivots"],
                                     None if cycled else r["rhs"], None if cycled else r["vrow"]))
        return out
    return evaluate


def host_search(jm: dict, width: int, depth, max_nodes: int = 10000, wave: int = 64):
    from oracle import iis as oracle_iis
    p = O.Problem(jm)
    log: list = []
    test = conflict.Tests(oracle_evaluate(p, log), max_nodes, depth, wave)
    _, support, relaxation = oracle_iis.start_set(p.M, p.vrow, p.vcol, p.unres, p.precision)
    return conflict.search(test, p.rows, p.ints, relaxation, support, width), test, log


def same_witness(a, b) -> bool:
    if a is None or b is None:
        return a is None and b is None
    return np.array_equal(a.rhs, b["rhs"]) and np.array_equal(np.asarray(a.vrow, dtype=np.int64), b["vrow"])


@pytest.mark.parametrize("case", ["example", "berlin_parity", "berlin_infeasible", "knapsack5", "random0", "planted(12, 10, 3, 2)"])
@pytest.mark.parametrize("width, depth", [(1, 1), (2, 3), (7, 16), (64, None), (1, None), (64, 1)])
def test_host_search_matches_the_restatement(case, width, depth):
    jm = CASES[case]()
    lit = O.conflict(jm)
    got, test, log = host_search(jm, width, depth)
    assert got["rows"] == lit["rows"] and got["ints"] == lit["ints"] and got["irreducible"] == lit["irreducible"]
    assert set(got["row_witness"]) == set(lit["row_witness"]) and set(got["int_witness"]) == set(lit["int_witness"])
    for r, w in lit["row_witness"].items():
        assert same_witness(got["row_witness"][r], w)
    for j, w in lit["int_witness"].items():
        assert same_witness(got["int_witness"][j], w)
    assert test.count["lps"] == sum(log) >= test.count["nodes"] and test.count["calls"] == len(log)


def test_depth_one_evaluates_only_committed_nodes():
    """With depth 1 every evaluated node is committed: speculation is the only source of extra LPs."""
    jm = problems.planted_integer_conflict_model(12, 10, 3, 2)
    _, test, _ = host_search(jm, 1, 1)
    assert test.count["lps"] == test.count["nodes"]


def test_searches_match_the_literal_dfs_node_for_node():
    """run() gives each test the literal search's verdict, witness and node count, at any depth."""
    jm = problems.planted_integer_conflict_model(12, 10, 3, 2)
    p = O.Problem(jm)
    tests = [(p.rows, p.ints), (p.rows, p.ints[:1]), ([r for r in p.rows if r > 2], p.ints), (p.rows[1:], p.ints)]
    for depth, max_nodes in itertools.product((1, 3, 16, None), (1, 2, 5, 10000)):
        out, count = conflict.run(oracle_evaluate(p, []), tests, max_nodes, depth, wave=8)
        total = 0
        for (rows, J), (v, w) in zip(tests, out):
            lv, lw, ln = O.test(p, rows, J, max_nodes)
            assert v == lv and same_witness(w, lw)
            total += ln
        assert count["nodes"] == total


def test_max_nodes_leaves_the_whole_model_undecided():
    jm = problems.planted_integer_conflict_model(12, 10, 3, 2)
    assert O.conflict(jm, max_nodes=2)["verdict"] == O.UNDECIDED
    with pytest.raises(ValueError, match="undecided within max_nodes"):
        host_search(jm, 4, None, max_nodes=2)


def test_a_model_with_a_plan_is_refused():
    jm = dict(EXAMPLE, constraints={"pair": {"equal": 4}, "cap": {"max": 1}})
    assert O.conflict(jm)["verdict"] == O.FEASIBLE
    with pytest.raises(ValueError, match="has an integer plan"):
        host_search(jm, 4, None)


# ---- front end ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model, kw, match", [
    ({**EXAMPLE, "ints": {}}, {}, r"Solve\(model, full=True\)\.iis\(\)"),
    ({**EXAMPLE, "constraints": {"pair": {"equal": 3, "weight": 2}}}, {}, "soft constraints"),
    ({**EXAMPLE, "constraints": {"pair": {"equal": 3, "priority": 1}}}, {}, "soft constraints"),
    ({**EXAMPLE, "optimize": {"cost": "min", "pair": "max"}}, {}, "one objective"),
    ({**EXAMPLE, "external": {"solver": "lpsolve"}}, {}, "external"),
    (EXAMPLE, {"max_nodes": 0}, "max_nodes= must be >= 1"),
    (EXAMPLE, {"width": 0}, "width= must be >= 1"),
    (EXAMPLE, {"depth": 1.5}, "depth= takes an integer"),
    ([], {}, "requires a model"),
    ("model", {}, "takes a JSON model"),
])
def test_conflict_refusals(model, kw, match):
    import jslpsolver_b200 as J
    with pytest.raises(ValueError, match=match):
        J.Conflict(model, **kw)


def test_solution_iis_still_refuses_mips():
    from jslpsolver_b200 import iis

    class _M:
        def getNumberOfIntegerVariables(self):
            return 1

    class _S:
        _tableau = type("T", (), {"model": _M()})()

    with pytest.raises(ValueError, match="integer or binary variables"):
        iis._check(_S())


# ---- C ABI --------------------------------------------------------------------------------------------------------
def _types(name):
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", header)
    assert proto, f"{name} is not declared"
    params = [p.strip() for p in proto.group(1).split(",")]
    return [re.sub(r"\s+", " ", p.rsplit("*", 1)[0]).strip() + " *" if "*" in p else p.rsplit(" ", 1)[0]
            for p in params]


def test_conflict_batch_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    C, P = _lib.C, _lib.C.c_void_p
    want = ["jslp_tab *", "const uint8_t *", "const uint8_t *", "const jslp_cut *", "const int32_t *", "int", "int",
            "int32_t *", "int32_t *", "int32_t *", "double *", "int32_t *", "double *", "int32_t *"]
    assert _types("jslp_conflict_batch") == want
    (_, res, got), = [s for s in _lib.SYMBOLS if s[0] == "jslp_conflict_batch"]
    assert res is C.c_int and got == [P] * 5 + [C.c_int] * 2 + [P] * 7

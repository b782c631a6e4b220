"""The MIP conflict on the H100 (DESIGN.md section 2n) against the sequential restatement in tests/conflict_oracle.py:
jslp_conflict_batch node by node (status, pivots, integrality, branching choice, final column 0 bits and labels)
through the node kernel and the single-tableau path, at the edges of both (empty and full keep sets, an empty integer
mask, cut counts at the shared-memory limit, log-cap overflow, cycling phase 1), and Conflict() on every model of the
CPU suite and on a planted conflict beyond shared memory, at several widths and depths."""
from __future__ import annotations

import json

import numpy as np
import pytest

import conflict_oracle as O
from conftest import load_bundle
from jslpsolver_b200 import _lib, problems
from test_conflict_cpu import CASES, check_conflict

pytestmark = pytest.mark.gpu


def bits(x) -> int:
    return int(np.float64(x).view(np.uint64))


def _gpu(jm: dict, engine=None, options=None):
    from jslpsolver_b200.model import Model
    from jslpsolver_b200.tableau import GpuTableau
    m = Model().loadJson(jm)
    g = GpuTableau(m.precision)
    g.setModel(m)
    if engine is not None:
        g.set_option(_lib.OPT_ENGINE, engine)
    for k, v in (options or {}).items():
        g.set_option(k, v)
    g.save()
    return g


def check_batch(jm: dict, specs: list, engine=None, options=None, what: str = "") -> dict:
    """jslp_conflict_batch over specs = [(rows, labels, cuts), ...] equals node() node by node; the tab is
    byte-identical afterwards."""
    p = O.Problem(jm)
    g = _gpu(jm, engine, options)
    H = p.M.shape[0]
    pos = {lab: i for i, lab in enumerate(p.ints)}
    keep = np.zeros((len(specs), H), dtype=np.uint8)
    int_keep = np.zeros((len(specs), len(p.ints)), dtype=np.uint8)
    for i, (rows, J, _) in enumerate(specs):
        keep[i, list(rows)] = 1
        int_keep[i, [pos[j] for j in J]] = 1
    before = (g.matrix2d().copy(), g.varIndexByRow.copy(), g.varIndexByCol.copy())
    res = g.conflict_batch(keep, int_keep, [c for _, _, c in specs])
    after = (g.matrix2d(), g.varIndexByRow, g.varIndexByCol)
    for a, b in zip(before, after):
        assert a.tobytes() == b.tobytes(), f"{what}: the tab changed"
    g.close()
    for i, (rows, J, cuts) in enumerate(specs):
        w = O.node(p, rows, J, cuts)
        tag = f"{what} node {i} ({len(rows)} rows, {len(J)} labels, {len(cuts)} cuts)"
        assert int(res["status"][i]) == w["status"], (tag, int(res["status"][i]), w["status"])
        assert int(res["pivots"][i]) == w["pivots"], (tag, int(res["pivots"][i]), w["pivots"])
        assert bool(res["is_integral"][i]) == w["is_integral"], tag
        assert int(res["branch_var"][i]) == w["branch_var"], tag
        assert bits(res["branch_value"][i]) == bits(w["branch_value"]), tag
        if w["status"] != O.UNDECIDED:
            h = len(w["vrow"])
            assert res["rhs"][i, :h].tobytes() == w["rhs"].tobytes(), tag
            assert np.array_equal(res["vrow"][i, :h], w["vrow"]), tag
    return res


def random_specs(p: O.Problem, n: int, seed: int, max_cuts: int = 4, keep: float = 0.85) -> list:
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        rows = [r for r in p.rows if rng.random() < keep]
        J = [j for j in p.ints if rng.random() < 0.7]
        cuts = [(int(rng.integers(0, 2)), int(p.ints[int(rng.integers(0, len(p.ints)))]), float(rng.integers(0, 4)))
                for _ in range(int(rng.integers(0, max_cuts + 1)))]
        out.append((rows, J, cuts))
    return out


BATCH_MODELS = {
    "example": CASES["example"],
    "planted 30x40": lambda: problems.planted_integer_conflict_model(30, 40, 4, 3),
    "knapsack 12x3": lambda: problems.knapsack_mip_model(12, 3, seed=4),
    "sudoku clue": CASES["sudoku"],
    "random mip 20x15": lambda: problems.random_mip_model(20, 15, seed=5),
}


@pytest.mark.parametrize("engine", [None, 2])
@pytest.mark.parametrize("name", list(BATCH_MODELS))
def test_conflict_batch_equals_the_restatement_node_by_node(name, engine):
    jm = BATCH_MODELS[name]()
    p = O.Problem(jm)
    specs = random_specs(p, 40 if engine is None else 10, 7)
    specs[0] = ([], list(p.ints), [])                      # an empty keep set
    specs[1] = (list(p.rows), list(p.ints), [])             # every row
    specs[2] = (list(p.rows), [], [])                       # an empty integer mask
    specs[3] = ([], list(p.ints), specs[3][2] or [(1, p.ints[0], 0.0)])  # cut rows only
    res = check_batch(jm, specs, engine, what=f"{name} engine {engine}")
    assert (res["status"] == 0).any()


def _smem_height_limit(W: int) -> int:
    """The tallest tableau of width W one node CTA holds (node_smem_bytes, with 4 KB kept free)."""
    import torch
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    ws = (W + 1) & ~1
    H = 1
    while 8 * ((H + 1) * ws + 2 * ws + H + 2) + 16 * (H + 1) + 4 * (2 * (H + 1) + W) + 16 <= optin - 4096:
        H += 1
    return H


@pytest.mark.parametrize("over", [0, 1])
def test_cut_counts_at_the_shared_memory_limit(over):
    """Kept rows plus cuts exactly at the node kernel's limit, and one cut row beyond it (the single-tableau path)."""
    jm = problems.planted_integer_conflict_model(60, 40, 3, 11)
    p = O.Problem(jm)
    nc = _smem_height_limit(p.M.shape[1]) - p.M.shape[0] + over
    rng = np.random.default_rng(over)
    specs = []
    for k in range(3):
        cuts = [(int(rng.integers(0, 2)), int(p.ints[int(rng.integers(0, len(p.ints)))]), float(rng.integers(0, 6)))
                for _ in range(nc)]
        specs.append((list(p.rows), list(p.ints), cuts))
    check_batch(jm, specs, what=f"{nc} cuts")


def test_log_cap_overflow_reruns_on_the_single_tableau_path():
    jm = problems.planted_integer_conflict_model(30, 40, 4, 3)
    p = O.Problem(jm)
    check_batch(jm, random_specs(p, 16, 9), options={_lib.OPT_NODE_LOG_CAP: 4}, what="log cap 4")


@pytest.mark.parametrize("engine", [None, 2])
def test_cycling_phase_one_is_a_cycled_node(engine):
    """ChenhuaWANG22_2's phase 1 cycles on the whole LP and on most one-row-smaller subsets (as in the IIS tests); with
    its variables made integer the node LPs must report the same cycles, stopped at the same pivot."""
    b = load_bundle()
    jm = json.loads(json.dumps([f for f in b["fixtures"] if f["file"] == "ChenhuaWANG22_2.json"][0]["model"]))
    jm["ints"] = {v: 1 for v in jm["variables"]}
    p = O.Problem(jm)
    specs = [(list(p.rows), list(p.ints), [])] + [([r for r in p.rows if r != s], list(p.ints), []) for s in p.rows]
    specs += [(list(p.rows), list(p.ints), [(1, p.ints[0], 0.0)])]
    res = check_batch(jm, specs, engine, what="ChenhuaWANG22_2")
    assert (res["status"] == 2).sum() >= 10


# ---- Conflict() -----------------------------------------------------------------------------------------------------
def _counters_removed(out: dict) -> dict:
    return {k: v for k, v in out.items() if k not in ("tests", "nodes", "lps", "launches", "pivots")}


@pytest.mark.parametrize("width, depth", [(1, 1), (8, None), (None, 1), (None, None)])
@pytest.mark.parametrize("case", list(CASES))
def test_conflict_equals_the_restatement(case, width, depth):
    import jslpsolver_b200 as J
    jm = CASES[case]()
    lit = O.conflict(jm)
    check_conflict(lit)
    got = J.Conflict(jm, width=width, depth=depth)
    assert _counters_removed(got) == O.named(lit)
    assert got["lps"] >= got["nodes"] >= got["tests"] > 0 and got["launches"] > 0


@pytest.mark.parametrize("engine", [2])
def test_conflict_on_the_single_tableau_path(engine):
    import jslpsolver_b200 as J
    s = J.Solver()
    s.engine = engine
    for case in ("example", "knapsack5", "planted(12, 10, 3, 2)"):
        jm = CASES[case]()
        assert _counters_removed(s.Conflict(jm)) == O.named(O.conflict(jm)), case


@pytest.mark.parametrize("width, depth", [(None, None), (8, 1)])
def test_planted_conflict_beyond_shared_memory(width, depth):
    import jslpsolver_b200 as J
    jm = problems.planted_integer_conflict_model(80, 400, 3, 5)
    got = J.Conflict(jm, width=width, depth=depth)
    assert _counters_removed(got) == O.named(O.conflict(jm))
    planted = sorted(v for v, coefs in jm["variables"].items() if "parity" in coefs)
    assert [c["name"] for c in got["constraints"]] == ["parity", "parity"]
    assert sorted(i["variable"] for i in got["integers"]) == planted

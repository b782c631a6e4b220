"""Near-optimal variability of a MIP on the H100 (DESIGN.md section 2o) against the sequential restatement in
tests/mip_variability_oracle.py: Variability() on every MIP fixture of the bundle through the node kernel and through
the single-tableau path (engine 2), values, witnesses and counters included; jslp_target_batch node by node (status,
evaluation bits, integrality, branching choice, pivots, final column 0 bits and labels) on bound tableaux of seeded
random MIPs, across launches, with resident and too-tall nodes mixed, with the log cap overflowing, and on a cycling
node; and one model beyond shared memory."""
from __future__ import annotations

import numpy as np
import pytest

import mip_variability_oracle as MO
import near_optimal_oracle as NO
import pool_oracle as PO
from jslpsolver_b200 import _lib, problems
from test_gpu_pool import beale_mip, bits, mip_fixtures

pytestmark = pytest.mark.gpu

COUNTERS = ("optimum", "allowance", "unique", "exact", "searches", "nodes", "lps", "rounds", "pivots")


def assert_same_report(got: dict, want: dict, what: str):
    for k in COUNTERS:
        assert got[k] == want[k], (what, k, got[k], want[k])
    assert got["variables"] == want["variables"], what
    assert got["constraints"] == want["constraints"], what


def call_both(jm: dict, engine: int, **kw):
    """(Variability() on the device, the restatement) or the two refusal messages."""
    import jslpsolver_b200 as J
    s = J.Solver()
    s.engine = engine
    try:
        want = MO.variability(jm, **kw)
    except ValueError as e:
        with pytest.raises(ValueError) as got:
            s.Variability(jm, **kw)
        assert str(got.value) == str(e)
        return None, None
    return s.Variability(jm, **kw), want


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("jm", [m for m in mip_fixtures() if len(m["variables"]) <= 200],
                         ids=lambda m: m.get("name") or str(len(m["variables"])))
def test_variability_equals_the_restatement_on_every_mip_fixture(jm, engine):
    for kw in ({"width": 4}, {"gap": 0.05, "width": 16, "points": True}):
        got, want = call_both(jm, engine, max_nodes=2000, **kw)
        if got is not None:
            assert_same_report(got, want, f"engine {engine} {kw}")
            assert got["launches"] > 0


def test_beyond_shared_memory_with_a_variable_subset():
    from conftest import load_bundle
    jm = next(f["model"] for f in load_bundle()["fixtures"] if f["file"] == "Monster_II.json")
    ints = [v for v in jm["variables"] if (jm.get("ints") or {}).get(v) or (jm.get("binaries") or {}).get(v)]
    got, want = call_both(jm, 0, variables=ints[:2], constraints=[], max_nodes=300, width=8, points=True)
    assert got is not None and got["searches"] == 4
    assert_same_report(got, want, "Monster_II")


def bound_pair(jm: dict, t: float, engine: int = 0, options=None, solve: bool = True):
    """(device bound tableau with its snapshot saved, the oracle's (B, vrow', vcol'), the oracle Problem) of the root LP
    optimum of jm (of its initial tableau without solve) at allowance t, checked bit for bit against each other."""
    from jslpsolver_b200.model import Model
    from jslpsolver_b200.tableau import GpuTableau
    from oracle.ref_model import OracleTableau
    p = PO.Problem(jm)
    m = Model().loadJson(jm)
    g = GpuTableau(m.precision)
    g.engine = engine
    g.options.update(options or {})
    g.setModel(m)
    if solve:
        g.simplex()
    b = g.bound(t)
    g.close()
    b.save()
    o = OracleTableau(p.M, p.vrow, p.vcol, precision=p.m.precision, integers=p.ints, check_cycles=p.m.checkForCycles)
    if solve:
        o.simplex()
    H, W = p.M.shape
    B = NO.bound(o.matrix(), *o.maps(), t, NO.fresh_label(W + H - 2, W + H - 2))
    assert b.matrix2d().tobytes() == B[0].tobytes() and np.array_equal(b.varIndexByRow, B[1])
    return b, B, p


def random_nodes(p: PO.Problem, n: int, seed: int, max_cuts: int = 4) -> list:
    """n nodes ([(label, -sense)], cuts): a random target (any label of the model, either sense) and random cuts on
    integer labels."""
    rng = np.random.default_rng(seed)
    labels = [int(v) for v in p.vcol[1:]] + [int(v) for v in p.vrow[1:]]
    out = []
    for _ in range(n):
        lab, s = int(rng.choice(labels)), int(rng.choice([-1, 1]))
        cuts = [(int(rng.integers(0, 2)), int(rng.choice(p.ints)), float(rng.integers(0, 4)))
                for _ in range(int(rng.integers(0, max_cuts + 1)))]
        out.append(([(lab, float(-s))], cuts))
    return out


def assert_batch(b, B, p, nodes, what: str) -> dict:
    """jslp_target_batch over nodes = [([(label, difference), ...], cuts), ...] equals MO.node_lp node by node; the
    tab is byte-identical afterwards."""
    before = (b.matrix2d().copy(), b.varIndexByRow.copy(), b.varIndexByCol.copy())
    res = b.target_batch([([(1, lab, d) for lab, d in edits], cuts) for edits, cuts in nodes], check_cycles=True)
    after = (b.matrix2d(), b.varIndexByRow, b.varIndexByCol)
    for x, y in zip(before, after):
        assert x.tobytes() == y.tobytes(), f"{what}: the tab changed"
    for i, (edits, cuts) in enumerate(nodes):
        w = MO.node_lp(p, *B, edits, cuts)
        tag = f"{what} node {i} ({edits}, {len(cuts)} cuts)"
        assert int(res["status"][i]) == w["status"], (tag, int(res["status"][i]), w["status"])
        assert bits(res["evaluation"][i]) == bits(w["evaluation"]), (tag, res["evaluation"][i], w["evaluation"])
        assert bool(res["is_integral"][i]) == w["is_integral"], tag
        assert int(res["branch_var"][i]) == w["branch_var"], tag
        assert bits(res["branch_value"][i]) == bits(w["branch_value"]), tag
        if w["status"] != PO.CYCLED:
            assert int(res["pivots"][i]) == w["pivots"], (tag, int(res["pivots"][i]), w["pivots"])
        if w["is_integral"]:
            h = len(w["vrow"])
            assert res["rhs"][i, :h].tobytes() == w["rhs"].tobytes(), tag
            assert np.array_equal(res["vrow"][i, :h], w["vrow"]), tag
    return res


@pytest.mark.parametrize("engine", [0, 2])
def test_target_batch_equals_the_restatement_node_by_node(engine):
    for seed, jm in enumerate([problems.random_mip_model(10, 6, seed=11, integer_fraction=0.6),
                               problems.knapsack_mip_model(12, 3, seed=4), problems.half_tie_mip_model(12, group=4)]):
        b, B, p = bound_pair(jm, 1e4, engine)
        # random nodes, and targets with every integer variable held at 0: their optima are integral
        nodes = random_nodes(p, 60, seed) + [(e, [(1, lab, 0.0) for lab in p.ints]) for e, _ in random_nodes(p, 6, 9)]
        res = assert_batch(b, B, p, nodes, f"{jm['name']} engine {engine}")
        assert (res["status"] == 0).any() and res["is_integral"].any() and not res["is_integral"].all()
        b.close()


def test_target_batch_more_nodes_than_one_launch():
    b, B, p = bound_pair(problems.single_knapsack_model(10, seed=7), 20.0)
    assert_batch(b, B, p, random_nodes(p, 4100, 5), "two launches")  # beyond batch_chunk's 4096 of this height
    b.close()


def test_target_batch_mixes_resident_and_too_tall_nodes():
    b, B, p = bound_pair(problems.single_knapsack_model(10, seed=8), 20.0)
    nodes = random_nodes(p, 12, 6)
    nodes[3] = (nodes[3][0], [(1, p.ints[0], 5.0)] * 2500 + [(0, p.ints[1], 1.0)])  # beyond shared memory
    res = assert_batch(b, B, p, nodes, "resident + tall")
    assert res["status"][3] in (0, 1)
    b.close()


def test_target_batch_log_cap_overflow_reruns_on_the_single_tableau_path():
    jm = problems.knapsack_mip_model(60, 6, seed=2)
    b, B, p = bound_pair(jm, 50.0, options={_lib.OPT_NODE_LOG_CAP: 4})
    nodes = random_nodes(p, 24, 9, max_cuts=6)
    res = assert_batch(b, B, p, nodes, "log cap 4")
    assert (res["pivots"] > 4).any()  # those overflowed the in-kernel log and ran on the single-tableau path
    b.close()


def test_target_batch_cycling_node():
    """Beale's objective set by cost edits on the bound tableau of Beale's initial tableau: the bound row's slack starts
    at 1e6, so it never ties the degenerate rows, and the simplex cycles as on Beale's LP."""
    jm = beale_mip()
    b, B, p = bound_pair(jm, 1e6, solve=False)
    beale = [(v.index, jm["variables"][v.id]["cost"]) for v in p.m.variables]
    nodes = [(beale, []), (beale, [(1, p.ints[0], 0.0)]), (beale, [(0, p.ints[0], 1.0)])] + random_nodes(p, 8, 3)
    res = assert_batch(b, B, p, nodes, "Beale")
    b.close()
    assert list(res["status"][:3]) == [PO.CYCLED, PO.CYCLED, PO.OPTIMAL]


def test_width_changes_no_range_on_the_device():
    import jslpsolver_b200 as J
    from conftest import load_bundle
    jm = next(f["model"] for f in load_bundle()["fixtures"] if f["file"] == "Sudoku4x4.json")
    runs = [J.Variability(jm, gap=0.0, width=w) for w in (1, None, 256)]
    for r in runs[1:]:
        assert {k: (e["min"], e["max"]) for k, e in r["variables"].items()} == \
            {k: (e["min"], e["max"]) for k, e in runs[0]["variables"].items()}
    for e in runs[1]["variables"].values():
        assert abs(e["min"]) < 1e-9 and abs(e["max"] - 1.0) < 1e-9

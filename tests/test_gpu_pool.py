"""The solution pool on the H100 (DESIGN.md section 2m) against the sequential restatement in tests/pool_oracle.py:
Pool() on every MIP fixture of the bundle through the node kernel and through the single-tableau path (engine 2),
jslp_pool_batch region by region (status, evaluation bits, integrality, branching choice, pivots, final column 0 bits
and labels) at the edges of its paths, speculation widths, the tie order, and the limit and unbounded stops."""
from __future__ import annotations

import math

import numpy as np
import pytest

import pool_oracle as O
from jslpsolver_b200 import _lib, problems

pytestmark = pytest.mark.gpu


def bits(x) -> int:
    return int(np.float64(x).view(np.uint64))


def mip_fixtures():
    from conftest import load_bundle
    b = load_bundle()
    return [f["model"] for f in b["fixtures"] + b["readme"] if f["model"].get("ints") or f["model"].get("binaries")]


def cap_of(jm: dict) -> int:
    return 300 if len(jm["variables"]) > 200 else 2000


def assert_same_pool(got: dict, want: dict, what: str):
    assert got["stop"] == want["stop"] and got["nodes"] == want["nodes"], (what, got["stop"], want["stop"],
                                                                          got["nodes"], want["nodes"])
    assert len(got["solutions"]) == len(want["solutions"]), what
    for g, w in zip(got["solutions"], want["solutions"]):
        assert bits(g["result"]) == bits(w["result"]), (what, g["result"], w["result"])
        assert g["values"] == w["values"] and g["rank"] == w["rank"], what
    assert got["lps"] >= got["nodes"]


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("jm", mip_fixtures(), ids=lambda m: m.get("name") or str(len(m["variables"])))
def test_pool_equals_the_sequential_search_on_every_mip_fixture(jm, engine):
    import jslpsolver_b200 as J
    s = J.Solver()
    s.engine = engine
    cap = cap_of(jm)
    for kw in ({}, {"gap": 0.05}):
        got = s.Pool(jm, k=5, max_nodes=cap, **kw)
        want = O.pool(jm, k=5, max_nodes=cap, **kw)
        assert_same_pool(got, want, f"engine {engine} {kw}")
        if got["solutions"]:
            ref = J.Solve(dict(jm, options={**(jm.get("options") or {}), "presolve": False}))
            first = got["solutions"][0]["result"]
            assert math.isclose(first, ref["result"], rel_tol=1e-9, abs_tol=1e-9), (first, ref["result"])


def random_regions(p: O.Problem, n: int, seed: int, max_cuts: int = 4) -> list:
    """n regions: random fixings of some integer variables (values 0..2) and random min / max cuts on others."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        labs = list(p.ints)
        rng.shuffle(labs)
        nf = int(rng.integers(0, len(labs) + 1))
        fixings = [(p.col_of[l], float(rng.integers(0, 3))) for l in labs[:nf]]
        cuts = [(int(rng.integers(0, 2)), int(labs[int(rng.integers(nf, len(labs)))]), float(rng.integers(0, 4)))
                for _ in range(int(rng.integers(0, max_cuts + 1)))] if nf < len(labs) else []
        out.append((fixings, cuts))
    return out


def assert_batch(jm: dict, regions: list, engine: int = 0, options=None, what: str = "") -> dict:
    """jslp_pool_batch over `regions` equals region_lp region by region; the tab is byte-identical afterwards."""
    from jslpsolver_b200.model import Model
    from jslpsolver_b200.tableau import GpuTableau
    p = O.Problem(jm)
    m = Model().loadJson(jm)
    g = GpuTableau(m.precision)
    g.engine = engine
    g.options.update(options or {})
    g.setModel(m)
    g.save()
    before = (g.matrix2d().copy(), g.varIndexByRow.copy(), g.varIndexByCol.copy())
    res = g.pool_batch(regions)
    after = (g.matrix2d(), g.varIndexByRow, g.varIndexByCol)
    for a, b in zip(before, after):
        assert a.tobytes() == b.tobytes(), f"{what}: the tab changed"
    for i, (f, c) in enumerate(regions):
        w = O.region_lp(p, f, c)
        tag = f"{what} region {i} ({len(f)} fixings, {len(c)} cuts)"
        assert int(res["status"][i]) == w["status"], (tag, int(res["status"][i]), w["status"])
        assert bits(res["evaluation"][i]) == bits(w["evaluation"]), (tag, res["evaluation"][i], w["evaluation"])
        assert bool(res["is_integral"][i]) == w["is_integral"], tag
        assert int(res["branch_var"][i]) == w["branch_var"], tag
        assert bits(res["branch_value"][i]) == bits(w["branch_value"]), tag
        if w["status"] != O.CYCLED:
            assert int(res["pivots"][i]) == w["pivots"], (tag, int(res["pivots"][i]), w["pivots"])
        if w["is_integral"]:
            h = len(w["vrow"])
            assert res["rhs"][i, :h].tobytes() == w["rhs"].tobytes(), tag
            assert np.array_equal(res["vrow"][i, :h], w["vrow"]), tag
    g.close()
    return res


@pytest.mark.parametrize("engine", [0, 2])
def test_pool_batch_equals_the_restatement_region_by_region(engine):
    for seed, jm in enumerate([problems.half_tie_mip_model(12, group=4), problems.knapsack_mip_model(12, 3, seed=4),
                               problems.set_cover_model(10, 8, seed=3)]):
        p = O.Problem(jm)
        regions = random_regions(p, 40, seed)
        regions[0] = ([], [])                                             # no fixing, no cut
        regions[1] = ([(p.col_of[l], 1.0) for l in p.ints], [])          # every integer variable fixed
        res = assert_batch(jm, regions, engine, what=f"{jm['name']} engine {engine}")
        assert (res["status"] == 0).any() and (res["status"] == 1).any()


def test_pool_batch_more_regions_than_one_launch():
    jm = problems.single_knapsack_model(10, seed=7)
    p = O.Problem(jm)
    regions = random_regions(p, 4100, 5)  # more than batch_chunk's 4096 regions of this height
    assert_batch(jm, regions, what="two launches")


def test_pool_batch_mixes_resident_and_too_tall_regions():
    jm = problems.single_knapsack_model(10, seed=8)
    p = O.Problem(jm)
    regions = random_regions(p, 12, 6)
    lab = p.ints[0]
    regions[3] = ([], [(1, lab, 5.0)] * 2500 + [(0, p.ints[1], 1.0)])  # beyond shared memory: single-tableau path
    res = assert_batch(jm, regions, what="resident + tall")
    assert res["status"][3] in (0, 1)


def test_pool_batch_long_logs_and_log_cap():
    jm = problems.knapsack_mip_model(120, 8, seed=2)
    p = O.Problem(jm)
    regions = [([(p.col_of[l], 0.0) for l in p.ints[:m]], [(1, p.ints[m], 0.0)] if m % 2 else [])
               for m in range(0, 48, 3)]
    res = assert_batch(jm, regions, what="long logs")
    assert (res["pivots"] > 64).any()  # some logs outgrew the inline head
    res = assert_batch(jm, regions, options={_lib.OPT_NODE_LOG_CAP: 4}, what="log cap 4")
    assert (res["pivots"] > 4).any()   # those overflowed the in-kernel log and ran on the single-tableau path


def beale_mip() -> dict:
    """Beale's cycling LP as a JSON model (min -0.75 x0 + 20 x1 - 0.5 x2 + 6 x3 over three rows), x2 integer."""
    rows = {"r1": [0.25, -8, -1, 9], "r2": [0.5, -12, -0.5, 3], "r3": [0, 0, 1, 0]}
    cost = [-0.75, 20, -0.5, 6]
    variables = {f"x{j}": {"cost": cost[j], **{r: v[j] for r, v in rows.items() if v[j]}} for j in range(4)}
    return {"name": "BealeMIP", "optimize": "cost", "opType": "min", "variables": variables,
            "constraints": {"r1": {"max": 0}, "r2": {"max": 0}, "r3": {"max": 1}}, "ints": {"x2": 1}}


def test_pool_batch_cycling_region():
    jm = beale_mip()
    p = O.Problem(jm)
    regions = [([], []), ([(p.col_of[p.ints[0]], 0.0)], []), ([], [(1, p.ints[0], 0.0)])]
    assert [O.region_lp(p, f, c)["status"] for f, c in regions] == [O.CYCLED, O.OPTIMAL, O.CYCLED]
    res = assert_batch(jm, regions, what="Beale")
    assert O.CYCLED in list(res["status"])


@pytest.mark.parametrize("jm", [problems.knapsack_mip_model(14, 3, seed=3), problems.half_tie_mip_model(10, group=4),
                                problems.set_cover_model(12, 9, seed=5)], ids=lambda m: m["name"])
def test_speculation_width_never_changes_the_pool(jm):
    import jslpsolver_b200 as J
    want = O.pool(jm, k=12, gap=0.2)
    lps = []
    for width in (1, 4, 64):
        got = J.Pool(jm, k=12, gap=0.2, width=width)
        assert_same_pool(got, want, f"width {width}")
        lps.append(got["lps"])
    assert lps[0] <= lps[2]


def test_half_tie_model_pins_the_tie_order():
    import jslpsolver_b200 as J
    jm = problems.half_tie_mip_model(12, group=4, seed=9)
    want = O.pool(jm, k=40, absolute_gap=3.0)
    assert len(want["solutions"]) > 5 and len({s["result"] for s in want["solutions"]}) < len(want["solutions"])
    assert_same_pool(J.Pool(jm, k=40, absolute_gap=3.0), want, "half ties")


def test_limit_stop_is_the_sequential_prefix():
    import jslpsolver_b200 as J
    jm = problems.knapsack_mip_model(12, 2, seed=6)
    for cap in (1, 7, 40):
        want = O.pool(jm, k=50, absolute_gap=1e9, max_nodes=cap)
        assert want["stop"] == "limit"
        assert_same_pool(J.Pool(jm, k=50, absolute_gap=1e9, max_nodes=cap), want, f"max_nodes {cap}")


def test_unbounded_relaxation_stops_unbounded():
    import jslpsolver_b200 as J
    jm = {"optimize": "v", "opType": "max", "constraints": {"c": {"max": 10}},
          "variables": {"x": {"v": 1, "c": 1}, "y": {"v": 2, "c": -1}}, "ints": {"x": 1}}
    got = J.Pool(jm, k=3)
    assert got["stop"] == "unbounded" and got["solutions"] == []
    assert O.pool(jm, k=3)["stop"] == "unbounded"


def test_infeasible_model_is_exhausted_with_no_solution():
    import jslpsolver_b200 as J
    jm = {"optimize": "v", "opType": "max", "constraints": {"c": {"max": 1}, "d": {"min": 2}},
          "variables": {"x": {"v": 1, "c": 1, "d": 1}}, "ints": {"x": 1}}
    got = J.Pool(jm, k=3)
    assert got["stop"] == "exhausted" and got["solutions"] == [] and got["nodes"] == 1

"""The Pareto frontier of a two-objective MIP on the H100 (DESIGN.md section 2s) against the sequential restatement in
tests/frontier_mip_oracle.py: FrontierMIP() through the node kernel (engine 0) and the single-tableau path (engine 2) at
widths 1, 16 and the default wave, points, values, open boxes, stops and counters included, on the families of
tests/test_frontier_mip_cpu.py; every MIP fixture of up to 200 variables with two seeded integer objectives; a model
whose box tableau is beyond shared memory; the node log cap at 4; every stop; jslp_box_batch node by node (right-hand
side edits on basic and non-basic slacks mixed with cost edits and cuts, resident and too-tall nodes in one call, log
cap overflow, a cycling node) and its refusals; and after every call every derived tableau closed and an unrelated
tableau unchanged."""
from __future__ import annotations

import numpy as np
import pytest

import frontier_mip_oracle as FO
import pool_oracle as PO
from helpers import strip_timeouts
from jslpsolver_b200 import _lib, iis, problems
from jslpsolver_b200.tableau import default_context
from test_frontier_mip_cpu import EXAMPLE, FAMILIES, assignment, general_ints, knapsack, planted
from test_gpu_mip_variability import bound_pair
from test_gpu_pool import beale_mip, bits, mip_fixtures

pytestmark = pytest.mark.gpu

KEYS = ("feasible", "bounded", "stop", "exact", "objectives", "step", "points", "open", "searches", "nodes", "lps",
        "rounds", "pivots")
BY_NAME = {m["name"]: m for m in FAMILIES}


def default_wave(jm: dict):
    """The default width's wave of a tableau of jm on this device (lexicographic_mip.run_stage, FrontierMIP())."""
    n_ints = len([v for v in {**(jm.get("ints") or {}), **(jm.get("binaries") or {})}.values() if v])
    ctx = default_context()
    return lambda h, w: iis.wave_width(ctx, h + min(n_ints, 8), w)


def call_both(jm: dict, engine: int = 0, options=None, **kw):
    """(FrontierMIP() on the device, the restatement), or (None, None) after checking both refuse alike.  Every tableau
    the call derives or uploads is closed when it returns, and an unrelated tableau keeps its bits."""
    import jslpsolver_b200 as J
    from jslpsolver_b200.model import Model
    from jslpsolver_b200.tableau import GpuTableau
    other = Model().loadJson(problems.knapsack_mip_model(12, 3, seed=4))
    g = GpuTableau(other.precision)
    g.setModel(other)
    g.simplex()
    before = (g.matrix2d().copy(), g.varIndexByRow.copy(), g.varIndexByCol.copy())
    s = J.Solver()
    s.engine = engine
    s.options.update(options or {})
    made = []
    adopt, upload = GpuTableau._adopt, GpuTableau.upload

    def tracked(self, h):
        c = adopt(self, h)
        made.append(c)
        return c

    def uploaded(self, *a, **k):
        made.append(self)
        return upload(self, *a, **k)

    wave = default_wave(jm) if kw.get("width") is None else (lambda h, w: 1)
    try:
        try:
            want, _ = FO.frontier_mip(jm, wave=wave, **kw)
        except ValueError as e:
            with pytest.raises(ValueError) as got:
                s.FrontierMIP(jm, **kw)
            assert str(got.value) == str(e)
            return None, None
        GpuTableau._adopt, GpuTableau.upload = tracked, uploaded
        try:
            got = s.FrontierMIP(jm, **kw)
        finally:
            GpuTableau._adopt, GpuTableau.upload = adopt, upload
        assert made and all(c.handle is None for c in made), "a tableau of the call was left open"
        after = (g.matrix2d(), g.varIndexByRow, g.varIndexByCol)
        for x, y in zip(before, after):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), "an unrelated tableau changed"
    finally:
        g.close()
    return got, want


def assert_same(got: dict, want: dict, what: str):
    for k in KEYS:
        assert got[k] == want[k], (what, k, got[k], want[k])
    assert got["launches"] > 0, what


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("width", [1, 16, None])
@pytest.mark.parametrize("name", ["knapsack8-2", "assignment3-1", "cover6x8-1", "planted6x1", "planted4x2", "ints-1"])
def test_frontier_mip_equals_the_restatement_on_the_families(name, width, engine):
    got, want = call_both(BY_NAME[name], engine, width=width)
    assert_same(got, want, f"{name} engine {engine} width {width}")
    assert got["stop"] == "reached" and len(got["points"]) >= 2


def test_the_example_on_the_device():
    got, want = call_both(EXAMPLE, 0)
    assert_same(got, want, "example")
    assert [(p["objectives"]["g1"], p["objectives"]["g2"]) for p in got["points"]] == [(0, 4), (3, 3), (4, 0)]


def with_objectives(jm: dict, seed: int) -> dict:
    """jm with two seeded integer objectives over its integer variables, max then min."""
    rng = np.random.default_rng(seed)
    jm = strip_timeouts(jm)
    ints = {v for v in jm["variables"] if (jm.get("ints") or {}).get(v) or (jm.get("binaries") or {}).get(v)}
    variables = {}
    for vid, attrs in jm["variables"].items():
        attrs = {a: x for a, x in attrs.items() if a not in ("front1", "front2")}
        if vid in ints:
            attrs["front1"], attrs["front2"] = int(rng.integers(0, 10)), int(rng.integers(0, 10))
        variables[vid] = attrs
    return dict(jm, variables=variables, optimize={"front1": "max", "front2": "min"})


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("jm", [m for m in mip_fixtures() if len(m["variables"]) <= 200],
                         ids=lambda m: m.get("name") or str(len(m["variables"])))
def test_every_mip_fixture_with_two_integer_objectives(jm, engine):
    got, want = call_both(with_objectives(jm, 7), engine, width=16, max_nodes=500, max_points=12)
    if got is not None:
        assert_same(got, want, f"engine {engine}")


def tall_planted(k: int = 5, pad: int = 5000) -> dict:
    """planted(k) with `pad` slack rows, so that its box tableau is beyond shared memory."""
    jm = planted(k)
    cons = dict(jm["constraints"], **{f"pad{r}": {"max": 10 + r % 3} for r in range(pad)})
    variables = {vid: dict(a, **{f"pad{r}": 1 for r in range(pad) if r % k == int(vid.split("_")[1])})
                 for vid, a in jm["variables"].items()}
    return dict(jm, name="tall", constraints=cons, variables=variables)


def test_beyond_shared_memory():
    jm = tall_planted()
    got, want = call_both(jm, 0, width=4)
    H, W = PO.Problem(FO.FM.loads(jm, *FO.FM.objectives(jm))["box"]).M.shape
    assert default_wave(jm)(H, W) == 1, "the box tableau fits shared memory"
    assert_same(got, want, "tall")
    assert len(got["points"]) == 5


def test_log_cap_overflow_reruns_on_the_single_tableau_path():
    for name in ("knapsack10-3", "assignment4-2"):
        got, want = call_both(BY_NAME[name], 0, options={_lib.OPT_NODE_LOG_CAP: 4}, width=8)
        assert got["stop"] == "reached"
        assert_same(got, want, f"log cap 4 {name}")


INFEASIBLE = {"optimize": {"a": "max", "b": "min"}, "constraints": {"odd": {"equal": 3}},
              "variables": {"x": {"odd": 2, "a": 1, "b": 1}, "y": {"odd": 2, "a": 1}}, "ints": {"x": 1, "y": 1}}
ONE_POINT = {"optimize": {"a": "max", "b": "max"}, "constraints": {"c": {"max": 3}},
             "variables": {"x": {"c": 1, "a": 1, "b": 2}}, "ints": {"x": 1}}
UNBOUNDED = {"optimize": {"a": "max", "b": "min"}, "constraints": {"c": {"min": 1}},
             "variables": {"x": {"c": 1, "a": 1, "b": 1}, "y": {"c": 1, "a": 0, "b": 2}}, "ints": {"x": 1, "y": 1}}


def beale_two() -> dict:
    """Beale's cycling MIP with its cost as the first objective and x2 as the second."""
    jm = beale_mip()
    variables = {v: dict(a, second=1 if v == "x2" else 0) for v, a in jm["variables"].items()}
    return dict(jm, variables=variables, optimize={"cost": "min", "second": "max"}, ints={v: 1 for v in variables})


@pytest.mark.parametrize("jm, kw, stop", [
    (INFEASIBLE, {}, None), (ONE_POINT, {}, "reached"), (UNBOUNDED, {}, "unbounded"), (planted(8), {"max_points": 4},
                                                                                         "limit"),
    (planted(8), {"max_nodes": 5}, "limit"), (knapsack(12, 7), {"max_nodes": 40}, "limit"),
    (knapsack(12, 7), {"max_nodes": 10}, "raises"), (planted(6), {"step": 5}, "reached"),
    (beale_two(), {"step": 0.25}, "any")],
    ids=["infeasible", "one-point", "unbounded", "max-points", "max-nodes-box", "max-nodes-box2", "max-nodes-end",
         "coarse-step", "beale"])
def test_every_stop(jm, kw, stop):
    got, want = call_both(jm, 0, width=1 if "max_nodes" in kw else 4, **kw)
    if got is None:  # both refused alike: the node limit before an end's first integer plan
        assert stop in ("raises", "any")
        return
    assert_same(got, want, str(stop))
    if stop != "any":
        assert got["stop"] == stop


# ---- jslp_box_batch node by node ---------------------------------------------------------------------------------------
def slack_labels(p: PO.Problem) -> list:
    return [c.index for c in p.m.constraints]


def random_nodes(p: PO.Problem, vrow, n: int, seed: int, max_cuts: int = 4) -> list:
    """n nodes (edits, cuts): up to three right-hand-side edits on random slacks (basic or not in the snapshot with
    row labels vrow), then up to three cost edits on random labels, then random cuts on integer labels."""
    rng = np.random.default_rng(seed)
    slacks = slack_labels(p)
    labels = [v.index for v in p.m.variables] + slacks
    out = []
    for _ in range(n):
        ed = [(0, int(rng.choice(slacks)), float(rng.integers(-4, 5))) for _ in range(int(rng.integers(0, 4)))]
        ed += [(1, int(rng.choice(labels)), float(rng.integers(-3, 4))) for _ in range(int(rng.integers(0, 4)))]
        cuts = [(int(rng.integers(0, 2)), int(rng.choice(p.ints)), float(rng.integers(0, 4)))
                for _ in range(int(rng.integers(0, max_cuts + 1)))]
        out.append((ed, cuts))
    return out


def assert_batch(b, B, p, nodes, what: str) -> dict:
    """jslp_box_batch over nodes equals FO.box_node_lp on the snapshot node by node; the tab is byte-identical
    afterwards."""
    before = (b.matrix2d().copy(), b.varIndexByRow.copy(), b.varIndexByCol.copy())
    res = b.box_batch(nodes, check_cycles=True)
    after = (b.matrix2d(), b.varIndexByRow, b.varIndexByCol)
    for x, y in zip(before, after):
        assert x.tobytes() == y.tobytes(), f"{what}: the tab changed"
    for i, (edits, cuts) in enumerate(nodes):
        w = FO.box_node_lp(p, edits, cuts, tableau=B)
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
def test_box_batch_equals_the_restatement_node_by_node(engine):
    kinds = set()
    for seed, jm in enumerate([problems.knapsack_mip_model(12, 3, seed=4), problems.half_tie_mip_model(12, group=4),
                               assignment(3, 5), general_ints(3)]):
        b, B, p = bound_pair(jm, 1e4, engine)
        basic = {int(v) for v in B[1][1:]}
        kinds |= {s in basic for s in slack_labels(p)}
        # random nodes, and nodes with every integer variable held at 0: their optima are integral
        nodes = random_nodes(p, B[1], 60, seed) + [(e, [(1, lab, 0.0) for lab in p.ints])
                                                   for e, _ in random_nodes(p, B[1], 6, 9)]
        res = assert_batch(b, B, p, nodes, f"{jm.get('name')} engine {engine}")
        assert (res["status"] == 0).any() and (res["status"] == 1).any() and res["is_integral"].any()
        b.close()
    assert kinds == {True, False}, "right-hand-side edits on basic and on non-basic slacks"


def test_box_batch_mixes_resident_and_too_tall_nodes():
    b, B, p = bound_pair(problems.single_knapsack_model(10, seed=8), 20.0)
    nodes = random_nodes(p, B[1], 12, 6)
    nodes[3] = (nodes[3][0], [(1, p.ints[0], 5.0)] * 2500 + [(0, p.ints[1], 1.0)])  # beyond shared memory
    res = assert_batch(b, B, p, nodes, "resident + tall")
    assert res["status"][3] in (0, 1)
    b.close()


def test_box_batch_log_cap_overflow_reruns_on_the_single_tableau_path():
    jm = problems.knapsack_mip_model(60, 6, seed=2)
    b, B, p = bound_pair(jm, 50.0, options={_lib.OPT_NODE_LOG_CAP: 4})
    res = assert_batch(b, B, p, random_nodes(p, B[1], 24, 9, max_cuts=6), "log cap 4")
    assert (res["pivots"] > 4).any()
    b.close()


def test_box_batch_cycling_node():
    """Beale's objective set by cost edits on the bound tableau of Beale's initial tableau, after right-hand-side edits
    of the bound row (basic) that keep its slack far from the degenerate rows."""
    jm = beale_mip()
    b, B, p = bound_pair(jm, 1e6, solve=False)
    beale = [(1, v.index, jm["variables"][v.id]["cost"]) for v in p.m.variables]
    last = int(B[1][-1])
    nodes = [([(0, last, 5.0)] + beale, []), ([(0, last, -5.0)] + beale, [(1, p.ints[0], 0.0)]),
             ([(0, last, 0.0)] + beale, [(0, p.ints[0], 1.0)])]
    res = assert_batch(b, B, p, nodes, "Beale")
    b.close()
    assert list(res["status"][:3]) == [PO.CYCLED, PO.CYCLED, PO.OPTIMAL]


def test_box_batch_refusals():
    from jslpsolver_b200.model import Model
    from jslpsolver_b200.tableau import GpuTableau
    m = Model().loadJson(problems.knapsack_mip_model(8, 2, seed=1))
    g = GpuTableau(m.precision)
    g.setModel(m)
    lab, slack = m.variables[0].index, m.constraints[0].index
    try:
        with pytest.raises(_lib.JslpError, match=r"box_batch needs a snapshot \(jslp_save\)"):
            g.box_batch([([(0, slack, 1.0)], [])])
        g.save()
        with pytest.raises(_lib.JslpError, match=r"box_batch: edit kind must be 0 \(rhs\) or 1 \(cost\)"):
            g.box_batch([([(2, lab, 1.0)], [])])
        with pytest.raises(_lib.JslpError, match="box_batch: unknown constraint or variable index"):
            g.box_batch([([(0, 10 ** 6, 1.0)], [])])
        with pytest.raises(_lib.JslpError, match="box_batch: a node's right-hand-side edits come before its cost"):
            g.box_batch([([(1, lab, 1.0), (0, slack, 1.0)], [])])
        res = g.box_batch([([(0, slack, 1.0), (1, lab, 1.0)], [(1, lab, 0.0)])])  # and the tab still answers
        assert int(res["status"][0]) in (0, 1)
    finally:
        g.close()

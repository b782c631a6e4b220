"""Repair of an infeasible MIP on the H100 (DESIGN.md section 2r) against the sequential restatement in
tests/repair_mip_oracle.py: RepairMIP() through the node kernel (engine 0) and the single-tableau path (engine 2) at
widths 1, 16 and the default wave, plan, stage optima bits, stops and counters included, on the infeasible families
of tests/test_repair_mip_cpu.py; every MIP fixture of up to 200 variables, where V* = 0 and stage 2 is the MIP
optimum; Monster_II, whose elastic tableau exceeds shared memory; the node log cap at 4; every stop; and after every
call every derived tableau closed and an unrelated tableau unchanged."""
from __future__ import annotations

import numpy as np
import pytest

import repair_mip_oracle as RMO
from helpers import strip_timeouts
from jslpsolver_b200 import _lib, iis, problems
from jslpsolver_b200.tableau import default_context
from test_gpu_pool import beale_mip, mip_fixtures
from test_repair_mip_cpu import FAMILIES, KNAP20, PACK, unbounded_stage_two, with_ints

pytestmark = pytest.mark.gpu

KEYS = ("feasible", "violation", "constraints", "values", "result", "stop", "stages", "nodes", "lps", "rounds",
        "pivots")


def default_wave(jm: dict):
    """The default width's wave of a stage tableau of jm on this device (lexicographic_mip.run_stage)."""
    n_ints = len([v for v in {**(jm.get("ints") or {}), **(jm.get("binaries") or {})}.values() if v])
    ctx = default_context()
    return lambda h, w: iis.wave_width(ctx, h + min(n_ints, 8), w)


def call_both(jm: dict, engine: int = 0, options=None, weights=None, **kw):
    """(RepairMIP() on the device, the restatement), or (None, None) after checking both refuse alike.  Every tableau
    the call derives is closed when it returns, and an unrelated tableau keeps its bits."""
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
    adopt = GpuTableau._adopt

    def tracked(self, h):
        c = adopt(self, h)
        made.append(c)
        return c

    wave = default_wave(jm) if kw.get("width") is None else 1
    GpuTableau._adopt = tracked
    try:
        try:
            want, _ = RMO.repair_mip(jm, weights, wave=wave, **kw)
        except ValueError as e:
            with pytest.raises(ValueError) as got:
                s.RepairMIP(jm, weights, **kw)
            assert str(got.value) == str(e)
            return None, None
        got = s.RepairMIP(jm, weights, **kw)
        assert made and all(c.handle is None for c in made), "a derived tableau was left open"
        after = (g.matrix2d(), g.varIndexByRow, g.varIndexByCol)
        for x, y in zip(before, after):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), "an unrelated tableau changed"
    finally:
        GpuTableau._adopt = adopt
        g.close()
    return got, want


def assert_same(got: dict, want: dict, what: str):
    for k in KEYS:
        assert got[k] == want[k], (what, k, got[k], want[k])
    assert got["launches"] > 0, what


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("width", [1, 16, None])
@pytest.mark.parametrize("name", list(FAMILIES))
def test_repair_mip_equals_the_restatement_on_the_infeasible_families(name, width, engine):
    for kw in ({}, {"gap": 0.05}, {"objective": False}):
        got, want = call_both(FAMILIES[name], engine, width=width, **kw)
        assert_same(got, want, f"{name} engine {engine} width {width} {kw}")
        assert got["violation"] > 0.0


def test_weight_subsets_and_no_integer_plan():
    from test_conflict_cpu import EXAMPLE
    for jm, weights in ((EXAMPLE, {"cap": 1.0}), (FAMILIES["planted1"], {"parity": {"max": 3.0}}),
                        (FAMILIES["packing3"], {f"c{i}": 1.0 + i % 3 for i in range(8)}),
                        (FAMILIES["planted2"], {"parity": 2.0, "resource0": 1.0})):
        got, want = call_both(jm, 0, weights=weights, width=4)
        assert_same(got, want, str(weights))
    assert got is not None
    got, _ = call_both(EXAMPLE, 0, weights={"cap": 1.0}, width=4)
    assert (got["feasible"], got["stop"], got["values"]) == (False, "infeasible", None)


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("jm", [m for m in mip_fixtures() if len(m["variables"]) <= 200],
                         ids=lambda m: m.get("name") or str(len(m["variables"])))
def test_every_mip_fixture_repairs_to_its_optimum(jm, engine):
    import jslpsolver_b200 as J
    got, want = call_both(jm, engine, width=16, max_nodes=2000)
    if got is None:
        return
    assert_same(got, want, f"engine {engine}")
    if got["stop"] != "reached" or jm.get("tolerance"):  # LargeFarmMIP's stage 2 reaches the node limit
        return
    sol = J.Solve(dict(strip_timeouts(jm), options={"presolve": False}))
    if sol["feasible"]:
        assert abs(got["violation"]) <= 1e-9 and got["constraints"] == []
        assert abs(got["result"] - sol["result"]) <= 1e-6 * max(1.0, abs(sol["result"])), (got["result"], sol)


@pytest.mark.parametrize("jm, kw, stop", [
    (unbounded_stage_two(), {}, "unbounded"), (beale_mip(), {}, "cycled"), (PACK, {"max_nodes": 3}, "limit"),
    (PACK, {"max_nodes": 9}, "limit"), (KNAP20, {"max_nodes": 5}, "limit"), (KNAP20, {"max_nodes": 20}, "limit"),
    (with_ints(problems.infeasible_packing_model(20, 16, 4, seed=5)),
     {"max_nodes": 8}, None), (FAMILIES["example"], {}, "reached")],
    ids=["unbounded", "cycled", "limit1-3", "limit1-9", "limit2-5", "limit2-20", "limit1-raises", "reached"])
def test_every_stop(jm, kw, stop):
    got, want = call_both(jm, 0, width=4, **kw)
    if stop is None:  # the stage-1 limit before any integral node: both raised the same ValueError
        assert got is None
        return
    assert_same(got, want, stop)
    assert got["stop"] == stop


def test_beyond_shared_memory():
    from conftest import load_bundle
    jm = next(f["model"] for f in load_bundle()["fixtures"] if f["file"] == "Monster_II.json")
    got, want = call_both(jm, 0, width=8, max_nodes=2000)
    assert iis.wave_width(default_context(), got["stages"][0]["height"],
                          got["stages"][0]["width"]) == 1, "the elastic tableau fits shared memory"
    assert_same(got, want, "Monster_II")


def test_log_cap_overflow_reruns_on_the_single_tableau_path():
    for jm in (FAMILIES["packing5"], FAMILIES["planted2"]):
        for kw in ({"width": 8}, {"gap": 0.02, "width": 8}):
            got, want = call_both(jm, 0, options={_lib.OPT_NODE_LOG_CAP: 4}, **kw)
            assert got["stop"] == "reached"
            assert_same(got, want, f"log cap 4 {kw}")

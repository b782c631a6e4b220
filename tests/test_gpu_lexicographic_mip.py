"""Lexicographic objectives of a MIP on the H100 (DESIGN.md section 2q) against the sequential restatement in
tests/lexicographic_mip_oracle.py: LexicographicMIP() on every MIP fixture of the bundle with seeded extra objectives,
through the node kernel (engine 0) and the single-tableau path (engine 2), plan, level optima bits, kinds, stops and
counters included; Monster_II, whose level tableaux exceed shared memory; the node log cap at 4; the node limit at
level 1 and at a later level; and after every call every level tableau closed and an unrelated tableau unchanged."""
from __future__ import annotations

import numpy as np
import pytest

import lexicographic_mip_oracle as LMO
from jslpsolver_b200 import _lib, problems
from test_gpu_pool import beale_mip, mip_fixtures
from test_lexicographic_mip_cpu import POINT, UNBOUNDED_1, UNBOUNDED_2, INFEASIBLE, with_extra, zero_first

pytestmark = pytest.mark.gpu

KEYS = ("feasible", "bounded", "stop", "objectives", "values", "levels", "nodes", "lps", "rounds", "pivots")


def call_both(jm: dict, engine: int = 0, options=None, **kw):
    """(LexicographicMIP() on the device, the restatement), or (None, None) after checking both refuse alike.  Every
    level tableau the call derives is closed when it returns."""
    import jslpsolver_b200 as J
    from jslpsolver_b200.tableau import GpuTableau
    s = J.Solver()
    s.engine = engine
    s.options.update(options or {})
    made = []
    adopt = GpuTableau._adopt

    def tracked(self, h):
        c = adopt(self, h)
        made.append(c)
        return c

    GpuTableau._adopt = tracked
    try:
        try:
            want, _ = LMO.chain(jm, **kw)
        except ValueError as e:
            with pytest.raises(ValueError) as got:
                s.LexicographicMIP(jm, **kw)
            assert str(got.value) == str(e)
            return None, None
        got = s.LexicographicMIP(jm, **kw)
    finally:
        GpuTableau._adopt = adopt
    assert all(c.handle is None for c in made), "a level tableau was left open"
    return got, want


def assert_same(got: dict, want: dict, what: str):
    for k in KEYS:
        assert got[k] == want[k], (what, k, got[k], want[k])
    assert got["launches"] > 0 or got["lps"] == 0, what


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("jm", [m for m in mip_fixtures() if len(m["variables"]) <= 200] + [beale_mip()],
                         ids=lambda m: m.get("name") or str(len(m["variables"])))
def test_lexicographic_mip_equals_the_restatement_on_every_mip_fixture(jm, engine):
    for kw in ({"width": 4}, {"gap": 0.05, "width": 16}, {"absolute_gap": {"extra1": 2.0}, "width": 1}):
        got, want = call_both(with_extra(jm, ["min", "max"], seed=3), engine, max_nodes=2000, **kw)
        if got is not None:
            assert_same(got, want, f"engine {engine} {kw}")


KNAP20 = problems.knapsack_mip_model(20, 3, seed=4)
KNAP20_FIRST = dict(KNAP20, optimize={KNAP20["optimize"]: "max", "nothing": "min"})


@pytest.mark.parametrize("jm, kw", [(POINT, {}), (INFEASIBLE, {}), (UNBOUNDED_1, {}), (UNBOUNDED_2, {}),
                                    (zero_first(KNAP20), {"max_nodes": 5}), (zero_first(KNAP20), {"max_nodes": 20}),
                                    (KNAP20_FIRST, {"max_nodes": 5}), (KNAP20_FIRST, {}),
                                    (zero_first(KNAP20), {"gap": 0.01})],
                         ids=["point", "infeasible", "unbounded1", "unbounded2", "limit2-5", "limit2-20", "limit1",
                              "cycled", "face"])
def test_every_kind_and_stop(jm, kw):
    got, want = call_both(jm, 0, width=4, **kw)
    assert_same(got, want, jm.get("name", "zero first"))
    if "max_nodes" in kw:  # the limit keeps the best integral node the level evaluated: the optimum, 381
        assert got["stop"] == "limit" and got["levels"][-1]["optimum"] == 381.0


def test_level_one_is_solve_without_presolve():
    import jslpsolver_b200 as J
    for jm in [with_extra(m, ["max"], seed=1) for m in mip_fixtures() if len(m["variables"]) <= 60 and m.get("optimize")]:
        key = next(iter(jm["optimize"]))
        single = dict(jm, optimize=key, opType=jm["optimize"][key], options={"presolve": False})
        try:
            res = J.LexicographicMIP(jm, width=8, max_nodes=2000)
        except ValueError as e:  # Fancy Stock Cutting: level 1 needs more nodes than that
            assert "raise max_nodes" in str(e)
            continue
        want = J.Solve(single)
        assert abs(res["levels"][0]["optimum"] - want["result"]) <= 1e-8 * max(1.0, abs(want["result"])), jm["name"]


def test_beyond_shared_memory():
    from conftest import load_bundle
    jm = next(f["model"] for f in load_bundle()["fixtures"] if f["file"] == "Monster_II.json")
    got, want = call_both(with_extra(jm, ["max"], seed=3), 0, max_nodes=2000, width=8)
    assert got["stop"] == "reached" and got["levels"][1]["kind"] == "bound"
    assert_same(got, want, "Monster_II")


def test_log_cap_overflow_reruns_on_the_single_tableau_path():
    jm = with_extra(problems.knapsack_mip_model(30, 4, seed=2), ["min", "max"], seed=5)
    for kw in ({"width": 8}, {"gap": 0.02, "width": 8}):
        got, want = call_both(jm, 0, options={_lib.OPT_NODE_LOG_CAP: 4}, **kw)
        assert got["stop"] == "reached"
        assert_same(got, want, f"log cap 4 {kw}")


def test_widths_change_no_optimum_and_an_unrelated_tableau_is_untouched():
    import jslpsolver_b200 as J
    from jslpsolver_b200.model import Model
    from jslpsolver_b200.tableau import GpuTableau
    other = Model().loadJson(problems.knapsack_mip_model(12, 3, seed=4))
    g = GpuTableau(other.precision)
    g.setModel(other)
    g.simplex()
    g.save()
    before = (g.matrix2d().copy(), g.varIndexByRow.copy(), g.varIndexByCol.copy())
    jm = with_extra(problems.knapsack_mip_model(16, 3, seed=9), ["min", "max"], seed=2)
    runs = [J.LexicographicMIP(jm, gap=0.02, width=w) for w in (1, None, 64)]
    for r in runs[1:]:
        assert [lv["optimum"] for lv in r["levels"]] == [lv["optimum"] for lv in runs[0]["levels"]]
        assert r["values"] == runs[0]["values"]
    after = (g.matrix2d(), g.varIndexByRow, g.varIndexByCol)
    for x, y in zip(before, after):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()
    g.close()

"""GPU checks of what-if scenarios (DESIGN.md section 2e): every scenario of jslp_scenario_batch -- status, pivot counts,
final right-hand-side column bits and row labels -- equals the sequential device path (a fresh tableau per scenario:
updateRightHandSide / updateCost / simplex) and the oracle definition, on the shared-memory batch and on the fallback
path (a tableau beyond shared memory, engines 1 and 2, the log cap, cycling scenarios); Solution.scenarios() equals the
Model-API path and the oracle key for key; and every call leaves the caller's tableau, labels, pivot log, saved
snapshot, sensitivity() and model as they were."""
import hashlib
import types

import numpy as np
import pytest

from conftest import load_bundle
from helpers import strip_timeouts

pytestmark = pytest.mark.gpu
BUNDLE = load_bundle()
STATUS = {"optimal": 0, "infeasible": 1, "unbounded": 2, "cycled": 3}
SEEN = {k: 0 for k in STATUS}


def _soft(jm):
    return any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())


CONTINUOUS = [f for f in BUNDLE["fixtures"] if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"]))
              and isinstance(f["model"].get("optimize"), str)]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _tableau(it, engine=0, options=None):
    from jslpsolver_b200 import _lib
    from jslpsolver_b200.tableau import GpuTableau
    g = GpuTableau(1e-8)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, it.integerIndices, it.optionalCosts)
    g.set_option(_lib.OPT_ENGINE, engine)
    g.set_option(_lib.OPT_PIVOT_LOG_CAP, 1 << 20)
    for k, v in (options or {}).items():
        g.set_option(k, v)
    g.simplex()
    return g


def _sequential(it, engine, edits):
    """The sequential device path of one scenario on a fresh tableau: (status, p1, p2, rhs, vrow)."""
    g = _tableau(it, engine)
    for kind, index, d in edits:
        if kind == 0:
            g.updateRightHandSide(index, d)
        else:
            g.updateCost(index, d)
    g.simplex()
    st = g.lastStatus
    status = 3 if st.cycled else 1 if not st.feasible else 2 if not st.bounded else 0
    out = (status, st.phase1_pivots, st.phase2_pivots, g.rhs_column().copy(), g.varIndexByRow.copy())
    g.close()
    return out


def _oracle_sol(it, M, vrow, vcol):
    """An oracle/scenarios source of the solved tableau (M, labels) of initial tableau `it`."""
    unres = {i: True for i in np.nonzero(it.unrestricted)[0]} if it.unrestricted is not None else {}
    model = types.SimpleNamespace(precision=1e-8, unrestrictedVariables=unres, checkForCycles=True, isMinimization=True)
    return types.SimpleNamespace(model=model, tableau=types.SimpleNamespace(matrix=lambda: M, maps=lambda: (vrow, vcol)))


def _oracle(src, edits):
    from oracle import scenarios as OS
    st, tab = OS.run(src, edits)
    M, (vrow, _) = tab.matrix(), tab.maps()
    status = 3 if st.cyclePhase else 1 if not st.feasible else 2 if not st.bounded else 0
    return status, st.lastP1, st.lastP2, M[:, 0].copy(), vrow


def _state(g):
    g._cache.clear()
    h = hashlib.sha256()
    for a in (g.matrix2d(), g.varIndexByRow, g.varIndexByCol, g.pivot_log()):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest(), g.evaluation, g.feasible, g.bounded, g._version


def assert_batch(it, g, scenarios, engine=0, what="", sequential_every=1, oracle=True):
    """Runs the scenarios (lists of (kind, index, difference)) in one call and pins every one to the sequential device
    path (every `sequential_every`-th) and to the oracle; checks the caller's state is untouched."""
    before = _state(g)
    g.save()
    M0 = g.matrix2d().copy()
    src = _oracle_sol(it, M0, g.varIndexByRow.copy(), g.varIndexByCol.copy()) if oracle else None
    edits, offsets = [], [0]
    for sc in scenarios:
        edits += sc
        offsets.append(len(edits))
    out = g.scenario_batch(edits, offsets)
    assert _state(g) == before, f"{what}: the caller's tableau changed"
    for k, sc in enumerate(scenarios):
        got = (int(out["status"][k]), int(out["p1"][k]), int(out["p2"][k]), out["rhs"][k], out["vrow"][k])
        SEEN[[n for n, v in STATUS.items() if v == got[0]][0]] += 1
        refs = []
        if k % sequential_every == 0:
            refs.append(("sequential", _sequential(it, engine, sc)))
        if oracle:
            refs.append(("oracle", _oracle(src, sc)))
        for name, want in refs:
            assert got[:3] == tuple(int(x) for x in want[:3]), (what, k, name, got[:3], want[:3])
            assert np.array_equal(_bits(got[3]), _bits(want[3])), (what, k, name, "rhs bits")
            assert np.array_equal(got[4], want[4]), (what, k, name, "row labels")
    # a save() from before the call still restores
    g.pivot(*_some_pivot(g))
    g.restore()
    g._cache.clear()
    assert np.array_equal(_bits(g.matrix2d()), _bits(M0)), f"{what}: restore() after the call"
    return out


def _some_pivot(g):
    M = g.matrix2d()
    r, c = np.argwhere(np.abs(M[1:, 1:]) > 1e-3)[0]
    return int(r + 1), int(c + 1)


def _picks(g, it, rng, n):
    """n scenarios: +-10 % on the right-hand sides of a few binding rows and basic-slack rows and on the costs of a few
    basic and non-basic variables (tableau units), in random order within each kind."""
    g._cache.clear()
    M, vr, vc = g.matrix2d(), g.varIndexByRow, g.varIndexByCol
    H0, W0 = it.matrix.shape
    slack_row = {int(it.varIndexByRow[r]): r for r in range(1, H0)}
    var_col = {int(it.varIndexByCol[c]): c for c in range(1, W0)}
    binding = [int(v) for v in vc[1:] if int(v) in slack_row]
    loose = [int(v) for v in vr[1:] if int(v) in slack_row]
    basic = [int(v) for v in vr[1:] if int(v) in var_col]
    nonbasic = [int(v) for v in vc[1:] if int(v) in var_col]
    out = []
    for _ in range(n):
        sc = []
        for pool in (binding, loose):
            for lab in rng.choice(pool, size=min(len(pool), int(rng.integers(0, 4))), replace=False) if pool else []:
                sc.append((0, int(lab), float(it.matrix[slack_row[int(lab)], 0]) * rng.uniform(-0.1, 0.1)))
        for pool in (basic, nonbasic):
            for lab in rng.choice(pool, size=min(len(pool), int(rng.integers(0, 3))), replace=False) if pool else []:
                sc.append((1, int(lab), float(it.matrix[0, var_col[int(lab)]]) * rng.uniform(-0.1, 0.1)))
        out.append(sc)
    return out


def _seeded(kind, n, m, seed, free_every=0):
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    if kind == "dense":
        return problems.dense_packing_lp_tableau(n, m, seed)
    jm = problems.mixed_lp_model(n, m, seed)
    if free_every:
        jm["unrestricted"] = {v: 1 for k, v in enumerate(jm["variables"]) if k % free_every == 0}
    return Model().loadJson(jm).initial_tableau()


@pytest.mark.parametrize("case", ["dense 150x120", "mixed 60x40", "mixed 60x40 unrestricted"])
def test_seeded_k2_scenarios(case):
    kind, n, m, seed, free = {"dense 150x120": ("dense", 150, 120, 5, 0), "mixed 60x40": ("mixed", 60, 40, 14, 0),
                              "mixed 60x40 unrestricted": ("mixed", 60, 40, 56, 6)}[case]
    it = _seeded(kind, n, m, seed, free)
    g = _tableau(it)
    assert g.feasible and g.bounded
    rng = np.random.default_rng(seed)
    sc = _picks(g, it, rng, 12) + [[], [(0, int(it.varIndexByRow[1]), 0.0)]]
    sc.append(sorted(sc[0] + sc[0], key=lambda e: e[0]))  # the same edits twice: each applies in turn
    assert_batch(it, g, sc, what=case)
    g.close()


def test_more_scenarios_than_one_wave():
    """600 scenarios of a 121x151 LP (one CTA each; more than the co-resident CTAs of one wave), all against the
    oracle, every 50th against the sequential path as well."""
    it = _seeded("dense", 150, 120, 8)
    g = _tableau(it)
    out = assert_batch(it, g, _picks(g, it, np.random.default_rng(1), 600), what="600", sequential_every=50)
    assert len(out["status"]) == 600
    g.close()


@pytest.mark.parametrize("engine", [1, 2])
def test_k2_sized_lp_on_the_fallback_path(engine):
    it = _seeded("dense", 150, 120, 14)
    g = _tableau(it, engine)
    assert_batch(it, g, _picks(g, it, np.random.default_rng(engine), 10), engine=engine, what=f"engine {engine}")
    g.close()


def test_log_cap_overflow_goes_to_the_fallback_path():
    from jslpsolver_b200 import _lib
    it = _seeded("dense", 150, 120, 9)
    g = _tableau(it, 0, {_lib.OPT_NODE_LOG_CAP: 3})
    out = assert_batch(it, g, _picks(g, it, np.random.default_rng(3), 16), what="log cap 3")
    assert (out["p1"] + out["p2"] > 3).any(), "no scenario outgrew the log cap"
    g.close()


def test_lp_beyond_shared_memory():
    it = _seeded("dense", 550, 600, 11)
    g = _tableau(it)
    assert_batch(it, g, _picks(g, it, np.random.default_rng(4), 8), what="601x551")
    g.close()


def test_cycling_scenarios():
    """From an optimum where unrestricted basic variables are negative, the re-solve starts with phase-1 pivots; on
    this LP they cycle even without an edit, so the cycle check declares the scenario infeasible on every path."""
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    jm = problems.mixed_lp_model(13, 11, seed=300 + 40 * 3 + 27)
    jm["unrestricted"] = {v: 1 for k, v in enumerate(jm["variables"]) if k % 4 == 0}
    it = Model().loadJson(dict(jm, opType="max")).initial_tableau()
    g = _tableau(it)
    assert g.feasible and g.bounded
    before = SEEN["cycled"]
    for engine in (0, 2):
        g.set_option(1, engine)  # JSLP_OPT_ENGINE: the batch, then the fallback path
        assert_batch(it, g, [[]] + _picks(g, it, np.random.default_rng(5), 6), engine=engine, what=f"cycling {engine}")
    assert SEEN["cycled"] > before
    g.close()


def test_config3_dense_2000():
    """The 2001x2001 benchmark LP, a handful of scenarios, against the sequential path (the oracle takes minutes per
    re-solve at this size)."""
    it = _seeded("dense", 2000, 2000, 12345)
    g = _tableau(it)
    assert_batch(it, g, _picks(g, it, np.random.default_rng(6), 3) + [[]], what="config 3", oracle=False)
    g.close()


def _model_sequential(jm, spec):
    """The literal Model-API path: Solve the model, setRightHandSide / Equality.setRightHandSide / setCost, solve()
    again, shape as Solve()."""
    import jslpsolver_b200 as J
    from jslpsolver_b200.model import Equality
    s = J.Solver()
    m = s._instance(jm, None)
    m.solve()
    for name, value in (spec.get("rhs") or {}).items():
        rows = [c for c in m.constraints if (c.name if c.name is not None else c.index) == name]
        if isinstance(value, dict):
            for side, v in value.items():
                next(c for c in rows if c.isUpperBound == (side == "max")).setRightHandSide(v)
        elif len(rows) == 2:
            up, lo = sorted(rows, key=lambda c: not c.isUpperBound)
            Equality(up, lo).setRightHandSide(value)
        else:
            rows[0].setRightHandSide(value)
    for vid, value in (spec.get("cost") or {}).items():
        m.setCost(value, next(v for v in m.variables if v.id == vid))
    out = s._finish(m, m.solve(), False)
    m.tableau.close()
    return out


def _specs(jm, m, n, seed):
    rng = np.random.default_rng(seed)
    fixed = m.presolveResult.fixedVariables if m.presolveResult is not None else {}
    specs = []
    for _ in range(n):
        spec = {"rhs": {}, "cost": {}}
        for name, c in jm["constraints"].items():
            if rng.random() < 0.3:
                f = lambda x: float(x) * (1.0 + rng.uniform(-0.1, 0.1))  # noqa: E731
                if c.get("equal") is None and c.get("min") is not None and c.get("max") is not None:
                    spec["rhs"][name] = {"max": f(c["max"]), "min": f(c["min"])}
                else:
                    spec["rhs"][name] = f(c.get("equal", c.get("max", c.get("min"))))
        for v in m.variables:
            if v not in fixed and rng.random() < 0.3:
                spec["cost"][v.id] = float(v.cost) * (1.0 + rng.uniform(-0.1, 0.1)) + 0.5
        specs.append(spec)
    return specs


@pytest.mark.parametrize("fx", CONTINUOUS, ids=lambda f: f["file"])
def test_fixture_results_equal_the_model_api_path_and_the_oracle(fx):
    import jslpsolver_b200 as J
    from jslpsolver_b200.scenarios import edits_of
    from oracle import ref_model
    from oracle import scenarios as OS
    jm = strip_timeouts(fx["model"])
    sol = J.Solve(jm, full=True)
    if not (sol.feasible and sol.bounded):
        pytest.skip("no optimum")
    t, m = sol._tableau, sol._tableau.model
    n = 2 if len(jm["constraints"]) > 100 else 8
    specs = _specs(jm, m, n, seed=len(fx["file"])) + [{}]
    rhs0, cost0 = [c.rhs for c in m.constraints], [v.cost for v in m.variables]
    rep = sol.sensitivity()
    t.set_option(3, 1 << 20)  # JSLP_OPT_PIVOT_LOG_CAP
    before = _state(t)
    got = sol.scenarios(specs)
    assert _state(t) == before and sol.sensitivity() == rep
    assert [c.rhs for c in m.constraints] == rhs0 and [v.cost for v in m.variables] == cost0
    assert not any("Cycle" in str(x) for x in m.messages)
    osol = ref_model.solve_full(jm, fast_cycles=True)
    for spec, g in zip(specs, got):
        seq = _model_sequential(jm, spec)
        want = OS.result(osol, edits_of(m, spec))
        for name, ref in (("Model API", seq), ("oracle", want)):
            assert list(g) == list(ref) and all(np.float64(g[k]).tobytes() == np.float64(ref[k]).tobytes()
                                                for k in g if not isinstance(g[k], bool)), (fx["file"], name, spec, g, ref)
    assert got[-1] == J.Solve(jm)


def test_infeasible_unbounded_and_berlin_on_the_device():
    import jslpsolver_b200 as J
    jm = {"optimize": "z", "opType": "max", "constraints": {"a": {"max": 10}, "b": {"min": 2}},
          "variables": {"x": {"z": 1, "a": 1, "b": 1}, "y": {"z": -1}}}
    sol = J.Solve(jm, full=True)
    specs = [{"rhs": {"a": 1.5}}, {"cost": {"y": 0.5}}, {"rhs": {"a": 12}}, {}]
    got = sol.scenarios(specs)
    assert (got[0]["feasible"], got[0]["result"]) == (False, 10.0)
    assert (got[1]["feasible"], got[1]["bounded"], got[1]["result"]) == (True, False, float("inf"))
    assert got[2]["result"] == 12.0 and got[3] == J.Solve(jm)
    for spec, g in zip(specs, got):
        assert g == _model_sequential(jm, spec), spec
    berlin = {"optimize": "capacity", "opType": "max",
              "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
              "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                            "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}
    a, b, c = J.Solve(berlin, full=True).scenarios([{"rhs": {"person": 352}}, {"rhs": {"person": 0}},
                                                    {"cost": {"brit": 40000}}])
    assert a["result"] == 880000.0 and b["result"] == 0 and (c["result"], c["brit"]) == (1760000.0, 44.0)


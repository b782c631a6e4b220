"""GPU checks of the sensitivity report: jslp_sensitivity's bounds are bit-identical to oracle/sensitivity.py on the same
final tableau (after solves with the automatic engine, whose ping-pong step leaves the result in either buffer, and
with the two-kernel engine, which updates in place), the whole report equals the one built from the oracle's own solve,
the call leaves the tableau as it was, and the error cases raise."""
import hashlib

import numpy as np
import pytest

from conftest import load_bundle
from helpers import strip_timeouts

pytestmark = pytest.mark.gpu
BUNDLE = load_bundle()
ENGINES = {"auto": 0, "two_kernel": 1}


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _soft(jm):
    return any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())


def _solve(it, engine, precision=1e-8):
    from jslpsolver_b200 import _lib
    from jslpsolver_b200.tableau import GpuTableau
    g = GpuTableau(precision)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, it.integerIndices, it.optionalCosts)
    g.set_option(_lib.OPT_ENGINE, engine)
    g.simplex()
    return g


def assert_bounds_match(g, unrestricted, what):
    from oracle import sensitivity as S
    want = S.bounds(g.matrix2d(), g.varIndexByRow, g.varIndexByCol, unrestricted, g.precision)
    got = g.sensitivity_bounds()
    for name, a, b in zip(("col_lo", "col_hi", "row_lo", "row_hi"), got, want):
        assert a.shape == b.shape, (what, name)
        bad = np.nonzero(_bits(a) != _bits(b))[0]
        assert len(bad) == 0, f"{what}: {name} differs at {bad[:5].tolist()}: device {a[bad[:5]]} restatement {b[bad[:5]]}"


CONTINUOUS = [f for f in BUNDLE["fixtures"] if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"]))
              and isinstance(f["model"].get("optimize"), str)]


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("fx", CONTINUOUS, ids=lambda f: f["file"])
def test_fixture_bounds_bit_identical(fx, engine):
    from jslpsolver_b200.model import Model, presolve
    m = Model().loadJson(strip_timeouts(fx["model"]))
    pr = presolve(m)
    if pr.isInfeasible:
        pytest.skip("decided by presolve")
    for v in pr.fixedVariables:
        v.cost = 0
    it = m.initial_tableau()
    g = _solve(it, ENGINES[engine])
    assert_bounds_match(g, it.unrestricted, fx["file"])


def _with_unrestricted(jm, every):
    jm = dict(jm)
    jm["unrestricted"] = {v: 1 for k, v in enumerate(jm["variables"]) if k % every == 0}
    return jm


SEEDED = {"dense 5x4": ("dense", 5, 4, 1), "dense 64x64": ("dense", 64, 64, 3), "dense 333x257": ("dense", 333, 257, 5),
          "mixed 12x9": ("mixed", 12, 9, 11), "mixed 120x80": ("mixed", 120, 80, 13),
          "mixed 40x30 unrestricted": ("mixed_free", 40, 30, 12), "mixed 260x200 unrestricted": ("mixed_free", 260, 200, 14),
          "wide mixed 2100x30": ("mixed", 2100, 30, 15), "tall dense 40x10000": ("dense", 40, 10000, 8),
          "config 3 dense 2000x2000": ("dense", 2000, 2000, 12345),
          # k_sensitivity's partition edges: one 256-column block exactly and one column past it (W = 256, 257, 512,
          # 513), and H - 1 = 2112 / 2113 rows: 8-row warp groups x 264 row blocks end on / one row past a full pass
          "dense 255x40": ("dense", 255, 40, 21), "mixed 256x30": ("mixed", 256, 30, 22),
          "dense 511x24": ("dense", 511, 24, 23), "mixed 512x20": ("mixed", 512, 20, 24),
          "tall dense 20x2112": ("dense", 20, 2112, 25), "tall dense 20x2113": ("dense", 20, 2113, 26)}


def _seeded_tableau(kind, n, m, seed):
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    if kind == "dense":
        return problems.dense_packing_lp_tableau(n, m, seed)
    jm = problems.mixed_lp_model(n, m, seed)
    if kind == "mixed_free":
        jm = _with_unrestricted(jm, 4)
    return Model().loadJson(jm).initial_tableau()


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("case", list(SEEDED))
def test_seeded_bounds_bit_identical(case, engine):
    it = _seeded_tableau(*SEEDED[case])
    g = _solve(it, ENGINES[engine])
    if case.startswith("mixed") and "unrestricted" in case:
        assert it.unrestricted.any()
    assert_bounds_match(g, it.unrestricted, f"{case} [{engine}]")
    g.close()


REPORT_MODELS = [(f["file"], f["model"]) for f in CONTINUOUS + [r for r in BUNDLE["readme"] if not (
    r["model"].get("ints") or r["model"].get("binaries") or _soft(r["model"])) and isinstance(r["model"].get("optimize"), str)]]


def _extra_models():
    from jslpsolver_b200 import problems
    return [("dense 30x20", problems.dense_packing_lp_model(30, 20, seed=2)),
            ("mixed 40x30", problems.mixed_lp_model(40, 30, seed=12)),
            ("mixed 40x30 unrestricted", _with_unrestricted(problems.mixed_lp_model(40, 30, seed=18), 4)),
            ("mixed 14x10 unrestricted", _with_unrestricted(problems.mixed_lp_model(14, 10, seed=13), 5))]


@pytest.mark.parametrize("engine", list(ENGINES))
def test_report_equals_the_restatement(engine):
    """Solve(model, full=True).sensitivity() against the report built from the oracle's own solve: every key, value
    and row, compared exactly."""
    import jslpsolver_b200 as J
    from oracle import ref_model
    from oracle import sensitivity as S
    s = J.Solver()
    s.engine = ENGINES[engine]
    checked = 0
    for name, jm in REPORT_MODELS + _extra_models():
        jm = strip_timeouts(jm)
        osol = ref_model.solve_full(jm, fast_cycles=True)
        gsol = s.Solve(jm, full=True)
        if osol.tableau is None or not (osol.feasible and osol.bounded):
            with pytest.raises(ValueError):
                gsol.sensitivity()
            continue
        assert gsol.sensitivity() == S.report(jm, osol), name
        checked += 1
    assert checked >= 20, checked


def _state_hash(g):
    g._cache.clear()
    h = hashlib.sha256()
    for a in (g.matrix2d(), g.varIndexByRow, g.varIndexByCol):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def test_report_leaves_the_tableau_unchanged_and_edits_still_match():
    """sensitivity() changes neither the tableau nor its maps, and the next solve still follows the oracle's; after a right-hand-side edit and a re-solve the tableau and the bounds still equal the oracle's."""
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    from oracle import ref_model
    from oracle import sensitivity as S
    m = Model().loadJson(problems.mixed_lp_model(40, 30, seed=12))
    m.tableau.engine = 2  # the fused step, as the dynamic-modification parity tests run edits
    sol = m.solve()
    assert sol.feasible and sol.bounded
    it = m.initial_tableau()  # what was uploaded: after presolve, before any edit
    g = m.tableau
    before = _state_hash(g)
    rep = sol.sensitivity()
    assert _state_hash(g) == before
    assert sol.sensitivity() == rep
    o = ref_model.OracleTableau(it.matrix, it.varIndexByRow, it.varIndexByCol, unrestricted=it.unrestricted, fast_cycles=True)
    o.simplex()
    # the next simplex() runs as the oracle's does from the same state
    g.simplex()
    o.simplex()
    assert np.array_equal(_bits(g.matrix2d()), _bits(o.matrix())) and np.array_equal(g.varIndexByRow, o.maps()[0])
    con = next(c for c in m.constraints if c.index in set(int(v) for v in g.varIndexByCol[1:]))  # a binding row
    diff = 0.25 * (rep["constraints"][m.constraints.index(con)]["range"]["max"] - con.rhs)
    if not np.isfinite(diff):
        diff = 1.0
    old_rhs = con.rhs
    con.setRightHandSide(old_rhs + diff)
    with pytest.raises(ValueError, match="edited or solved again"):
        sol.sensitivity()
    d = con.rhs - old_rhs  # the difference Constraint.setRightHandSide hands the tableau
    o.update_rhs(con.index, -d if con.isUpperBound else d)
    sol2 = m.solve()
    o.simplex()
    assert np.array_equal(_bits(g.matrix2d()), _bits(o.matrix()))
    assert np.array_equal(g.varIndexByRow, o.maps()[0]) and np.array_equal(g.varIndexByCol, o.maps()[1])
    assert_bounds_match(g, it.unrestricted, "after updateRightHandSide")
    rep2 = sol2.sensitivity()
    assert rep2["constraints"][m.constraints.index(con)]["rhs"] == con.rhs
    want = S.bounds(o.matrix(), *o.maps(), it.unrestricted, g.precision)
    assert all(np.array_equal(_bits(a), _bits(b)) for a, b in zip(g.sensitivity_bounds(), want))


def test_error_cases_raise():
    import jslpsolver_b200 as J
    lp = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Berlin Air Lift Problem.json"][0]["model"])
    mip = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Integer Berlin Air Lift Problem.json"][0]["model"])
    with pytest.raises(ValueError, match="integer or binary"):
        J.Solve(mip, full=True).sensitivity()
    soft = dict(lp, constraints=dict(lp["constraints"], plane={"max": 30, "weight": 100}))
    with pytest.raises(ValueError, match="soft constraints"):
        J.Solve(soft, full=True).sensitivity()
    infeasible = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Infeasible Berlin Air Lift Problem.json"][0]["model"])
    with pytest.raises(ValueError, match="infeasible"):
        J.Solve(infeasible, full=True).sensitivity()
    unbounded = {"optimize": "z", "opType": "max", "constraints": {"c": {"min": 1}},
                 "variables": {"x": {"z": 1, "c": 1}}}
    sol = J.Solve(unbounded, full=True)
    assert not sol.bounded
    with pytest.raises(ValueError, match="unbounded"):
        sol.sensitivity()
    m = J.Model().loadJson(lp)
    first = m.solve()
    first.sensitivity()
    m.solve()  # solved again: the first solution no longer describes the tableau
    with pytest.raises(ValueError, match="edited or solved again"):
        first.sensitivity()

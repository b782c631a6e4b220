"""GPU checks of alternative optima (DESIGN.md section 2h): jslp_face_create against the NumPy restatement bit for bit
(W', map, vcol', vrow', every double of F with its +0 cost row) on solved fixtures and seeded LPs, on the 2001 x 2001
benchmark optimum and at the edges of the plan and gather kernels' geometry with threshold cost entries; every target
LP on the face (status, pivot counts, raw evaluation, column 0, row labels) against the oracle on the shared-memory
batch and on the single-tableau path; the parent tableau untouched; and Solution.variability() equal to the oracle's
end to end, with sensitivity() and scenarios() unchanged afterwards."""
import hashlib
import math

import numpy as np
import pytest

from conftest import load_bundle
from helpers import strip_timeouts

pytestmark = pytest.mark.gpu
BUNDLE = load_bundle()
P = 1e-8


def _soft(jm):
    return any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())


CONTINUOUS = [f for f in BUNDLE["fixtures"]
              if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"])
                      or f["model"].get("unrestricted"))
              and isinstance(f["model"].get("optimize"), str)]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _upload(M, vrow, vcol, engine=0, options=None):
    from jslpsolver_b200 import _lib
    from jslpsolver_b200.tableau import GpuTableau
    g = GpuTableau(P)
    g.upload(M, vrow, vcol)
    g.set_option(_lib.OPT_ENGINE, engine)
    g.set_option(_lib.OPT_PIVOT_LOG_CAP, 1 << 20)
    for k, v in (options or {}).items():
        g.set_option(k, v)
    return g


def _solved(it, engine=0, options=None):
    g = _upload(it.matrix, it.varIndexByRow, it.varIndexByCol, engine, options)
    g.simplex()
    assert g.feasible and g.bounded
    return g


def _state(g):
    g._cache.clear()
    h = hashlib.sha256()
    for a in (g.matrix2d(), g.varIndexByRow, g.varIndexByCol, g.pivot_log()):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest(), g.evaluation, g.feasible, g.bounded, g._version


def assert_face(g, what=""):
    """g.face() against oracle/variability.face on g's own tableau; returns (face or None, kept, F, vcol')."""
    from oracle import variability as OV
    before = _state(g)
    M, vrow, vcol = g.matrix2d().copy(), g.varIndexByRow.copy(), g.varIndexByCol.copy()
    kept, F, vcol_f = OV.face(M, vcol, P)
    f, got = g.face()
    assert np.array_equal(got, kept), (what, "map", got[:8], kept[:8], len(got), len(kept))
    assert _state(g) == before, f"{what}: the parent tableau changed"
    if len(kept) == 1:
        assert f is None, what
        return None, kept, F, vcol_f
    assert (f.height, f.width) == F.shape, what
    Fg = f.matrix2d()
    assert np.array_equal(_bits(Fg), _bits(F)), (what, "F bits", int((_bits(Fg) != _bits(F)).sum()))
    assert not np.signbit(Fg[0]).any() and (Fg[0] == 0).all(), (what, "row 0 is +0")
    assert np.array_equal(f.varIndexByCol[1:], vcol_f[1:]) and np.array_equal(f.varIndexByRow[1:], vrow[1:]), what
    info = (f.nVars, f.lastElementIndex)
    f._refresh_dims()
    assert (f.width, f.height, f.nVars, f.lastElementIndex) == (F.shape[1], F.shape[0]) + info == \
        (F.shape[1], F.shape[0], g.nVars, g.lastElementIndex), what
    return f, kept, F, vcol_f


def assert_targets(g, f, F, vcol_f, targets, what=""):
    """The (label, sense) targets as one scenario batch on the face against the oracle's rule 3."""
    from oracle import variability as OV
    vrow = g.varIndexByRow.copy()
    out = f.scenario_batch([(1, lab, float(-s)) for lab, s in targets], list(range(len(targets) + 1)), check_cycles=True)
    seen = set()
    for k, (lab, s) in enumerate(targets):
        status, ev, p1, p2, rhs, vr = OV.target(F, vrow, vcol_f, P, lab, s)
        got = (int(out["status"][k]), int(out["p1"][k]), int(out["p2"][k]))
        assert got == (status, p1, p2), (what, k, lab, s, got, (status, p1, p2))
        if status == 0:
            assert _bits(out["eval_raw"][k]) == _bits(ev), (what, k, "eval_raw", out["eval_raw"][k], ev)
        assert np.array_equal(_bits(out["rhs"][k]), _bits(rhs)), (what, k, "column 0 bits")
        assert np.array_equal(out["vrow"][k][1:], vr[1:]), (what, k, "row labels")
        seen.add(status)
    return seen


def _all_targets(g, kept):
    vrow, vcol = g.varIndexByRow, g.varIndexByCol
    t = []
    for lab in vrow[1:]:
        t += [(int(lab), -1), (int(lab), 1)]
    return t + [(int(vcol[c]), 1) for c in kept[1:]]


def _alt(n, m, seed, **kw):
    from jslpsolver_b200 import problems
    return problems.lp_tableau(*problems.alternative_optima_arrays(n, m, seed, **kw))


# ---------------------------------------------------------------- the face kernels
@pytest.mark.parametrize("case", ["alt 40x24", "alt 150x120", "dense 150x120", "alt 550x600"])
def test_face_of_seeded_optima(case):
    from jslpsolver_b200 import problems
    it = {"alt 40x24": lambda: _alt(40, 24, 3), "alt 150x120": lambda: _alt(150, 120, 12345),
          "dense 150x120": lambda: problems.dense_packing_lp_tableau(150, 120, 5),
          "alt 550x600": lambda: _alt(550, 600, 7)}[case]()
    for pingpong in (1, 0):  # the optimum can end in either buffer of the pair: the face reads whichever is current
        from jslpsolver_b200 import _lib
        g = _solved(it, 0, {_lib.OPT_PINGPONG: pingpong})
        f, kept, F, vcol_f = assert_face(g, f"{case} pingpong {pingpong}")
        if case.startswith("alt"):
            assert len(kept) >= 3, "the planted block leaves free columns"
        if f is not None:
            f.close()
        g.close()


def test_config3_optimum():
    """The 2001 x 2001 benchmark LP: the face of its optimum, and whatever targets it has on the device path it takes."""
    from jslpsolver_b200 import problems
    g = _solved(problems.dense_packing_lp_tableau(2000, 2000, 12345))
    f, kept, F, vcol_f = assert_face(g, "config 3")
    if f is not None:
        assert_targets(g, f, F, vcol_f, _all_targets(g, kept)[:6], "config 3")
        f.close()
    g.close()


def _crafted(H, W, keep, seed):
    """An H x W tableau (not solved: the face reads any tableau) whose cost row keeps exactly the columns of `keep`."""
    rng = np.random.default_rng(seed)
    M = rng.uniform(-9, 9, size=(H, W))
    M[0, 1:] = rng.choice([3.5, -2.25, 1e-7, -1e-7], size=W - 1)
    inside = [0.0, -0.0, P, -P, 1e-300, -5e-9]
    for k, c in enumerate(sorted(keep)):
        M[0, c] = inside[k % len(inside)]
    vrow = np.concatenate([[-1], np.arange(H - 1)]).astype(np.int32)
    vcol = np.concatenate([[-1], H - 1 + np.arange(W - 1)]).astype(np.int32)
    return M, vrow, vcol


@pytest.mark.parametrize("W", [2, 3, 16, 17, 31, 32, 33, 34, 511, 512, 513, 514, 1023, 1024, 1025, 1026, 2047, 2048,
                               2049, 2050, 4097])
def test_plan_edges(W):
    """Kept / banned boundaries at the warp (32), tile (512) and pass (2048) edges of k_face_plan, W' odd and even."""
    edges = [c for c in (1, 30, 31, 32, 33, 510, 511, 512, 513, 1022, 1023, 1024, 1025, 2046, 2047, 2048, 2049, 4095,
                         4096) if c < W]
    rng = np.random.default_rng(W)
    for variant in range(4):
        keep = set(edges[variant % 2::2]) | set(int(c) for c in rng.choice(np.arange(1, W), size=min(W - 1, 7 + variant)))
        if variant == 3:
            keep = keep - {max(keep)} if len(keep) % 2 else keep  # W' = 1 + |keep|: both parities occur over variants
        M, vrow, vcol = _crafted(5, W, keep, seed=W + variant)
        g = _upload(M, vrow, vcol)
        f, kept, _, _ = assert_face(g, f"W {W} variant {variant}")
        assert set(int(c) for c in kept[1:]) == keep
        if f is not None:
            f.close()
        g.close()


@pytest.mark.parametrize("H", [1, 2, 16, 17, 63, 64, 65, 128, 129, 200])
def test_gather_edges(H):
    """Row blocks of 64 and column tiles of 16 of k_face_gather: W' = 15, 16, 17 (stride 16, 16, 32) and 33."""
    for n_keep in (14, 15, 16, 32):
        W = 50
        keep = set(range(1, W))
        keep = set(sorted(keep)[::1][:n_keep]) if H % 2 else set(sorted(keep)[-n_keep:])
        M, vrow, vcol = _crafted(H, W, keep, seed=H * 100 + n_keep)
        g = _upload(M, vrow, vcol)
        f, kept, _, _ = assert_face(g, f"H {H} keep {n_keep}")
        assert len(kept) == n_keep + 1
        f.close()
        g.close()


def test_threshold_cost_entries_and_extremes():
    """Cost entries exactly +-P and +-0 keep the column, one ulp beyond +-P and NaN ban it; no kept column gives no
    face; a zero cost row keeps every column."""
    cost = [7.0, P, -P, 0.0, -0.0, np.nextafter(P, 1), np.nextafter(-P, -1), math.nan, 5.0, -5.0, 1e-300, math.inf,
            -math.inf]
    M, vrow, vcol = _crafted(9, len(cost), set(), seed=1)
    M[0] = cost
    M[3, 4], M[4, 4] = -0.0, math.nan  # body values travel bit for bit
    g = _upload(M, vrow, vcol)
    f, kept, _, _ = assert_face(g, "thresholds")
    assert list(kept) == [0, 1, 2, 3, 4, 10]
    f.close()
    g.close()
    M, vrow, vcol = _crafted(9, 40, set(), seed=2)
    g = _upload(M, vrow, vcol)
    f, kept, _, _ = assert_face(g, "nothing kept")
    assert f is None and list(kept) == [0]
    g.close()
    M, vrow, vcol = _crafted(70, 1000, set(range(1, 1000)), seed=3)
    M[0, 1:] = 0.0
    g = _upload(M, vrow, vcol)
    f, kept, _, _ = assert_face(g, "everything kept")
    assert len(kept) == 1000
    f.close()
    g.close()


def test_optional_objectives_are_refused():
    from jslpsolver_b200._lib import JslpError
    from jslpsolver_b200.tableau import GpuTableau
    M, vrow, vcol = _crafted(4, 6, {1, 2}, seed=4)
    g = GpuTableau(P)
    g.upload(M, vrow, vcol, optionalCosts=np.ones((1, 6)))
    with pytest.raises(JslpError, match="optional objectives"):
        g.face()
    g.close()


# ---------------------------------------------------------------- the target LPs on the face
@pytest.mark.parametrize("engine", [0, 2])
def test_targets_match_the_oracle(engine):
    """Every target of two seeded optima with planted alternatives: engine 0 runs them one CTA each in shared memory,
    engine 2 one after another on the single-tableau path."""
    seen = set()
    for n, m, seed, kw in ((30, 16, 3, {}), (60, 40, 11, {"dup": 6, "par": 5})):
        g = _solved(_alt(n, m, seed, **kw), engine)
        f, kept, F, vcol_f = assert_face(g, f"alt {n}x{m}")
        before = _state(g)
        seen |= assert_targets(g, f, F, vcol_f, _all_targets(g, kept), f"alt {n}x{m} engine {engine}")
        assert _state(g) == before
        f.close()
        g.close()
    assert 0 in seen


def test_unbounded_face_on_the_device():
    """max x - y, x - y <= 2: both variables run off along the optimal ray."""
    import jslpsolver_b200 as J
    jm = {"optimize": "z", "opType": "max", "constraints": {"gap": {"max": 2}, "low": {"min": 1}},
          "variables": {"x": {"z": 1, "gap": 1, "low": 1}, "y": {"z": -1, "gap": -1}}}
    v = J.Solve(jm, full=True).variability(points=True)
    assert (v["variables"]["x"]["min"], v["variables"]["x"]["max"]) == (2.0, math.inf)
    assert (v["variables"]["y"]["min"], v["variables"]["y"]["max"]) == (0.0, math.inf)
    assert v["variables"]["y"]["argmax"] is None and v["variables"]["x"]["argmin"] == {"x": 2.0, "y": 0.0}
    assert v["exact"] and not v["unique"]


def test_face_beyond_shared_memory():
    """A 601 x 551 optimum with its cost row zeroed keeps every column: the face is as large as the tableau, beyond
    shared memory, so its targets run on the single-tableau path."""
    from jslpsolver_b200 import problems
    g0 = _solved(problems.dense_packing_lp_tableau(550, 600, 11))
    M, vrow, vcol = g0.matrix2d().copy(), g0.varIndexByRow.copy(), g0.varIndexByCol.copy()
    g0.close()
    M[0, 1:] = 0.0
    g = _upload(M, vrow, vcol)
    f, kept, F, vcol_f = assert_face(g, "601x551 all kept")
    assert len(kept) == 551
    basic = [int(x) for x in vrow[1:] if int(x) >= 600][:2]
    assert_targets(g, f, F, vcol_f, [(basic[0], 1), (basic[1], -1), (int(vcol[5]), 1)], "601x551")
    f.close()
    g.close()


# ---------------------------------------------------------------- Solution.variability() end to end
def _oracle_report(sol, points_of=None):
    """The report the oracle's ranges give for the device's own final tableau, shaped as the host shapes it."""
    from oracle import variability as OV
    t, m = sol._tableau, sol._tableau.model
    t._cache.clear()
    M, vrow, vcol = t.matrix2d().copy(), t.varIndexByRow.copy(), t.varIndexByCol.copy()
    fixed = m.presolveResult.fixedVariables if m.presolveResult is not None else {}
    labels = [v.index for v in m.variables if v not in fixed] + [c.index for c in m.constraints]
    want, free, lps, _ = OV.ranges(M, vrow, vcol, t.precision, labels)
    return want, free, lps, fixed


def assert_report(jm, what):
    import jslpsolver_b200 as J
    sol = J.Solve(jm, full=True)
    if not (sol.feasible and sol.bounded):
        return None
    t, m = sol._tableau, sol._tableau.model
    rep = sol.sensitivity()
    scen = sol.scenarios([{}])
    t.set_option(3, 1 << 20)  # JSLP_OPT_PIVOT_LOG_CAP
    before = _state(t)
    v = sol.variability(points=True)
    assert _state(t) == before, f"{what}: the caller's tableau changed"
    assert sol.sensitivity() == rep and sol.scenarios([{}]) == scen and sol.basis()
    assert not any("Cycle" in str(x) for x in m.messages)
    want, free, lps, fixed = _oracle_report(sol)
    assert (v["free"], v["lps"]) == (free, lps), (what, v["free"], v["lps"], free, lps)
    same = lambda a, b: (a is None and b is None) or (a is not None and b is not None and _bits(a) == _bits(b))  # noqa: E731
    for x in m.variables:
        e = v["variables"][x.id]
        if x in fixed:
            assert e["fixed"] and e["min"] == e["max"] == e["value"] == fixed[x]
            continue
        w = want[x.index]
        assert same(e["min"], w["min"]) and same(e["max"], w["max"]) and same(e["value"], w["value"]), (what, x.id, e, w)
        for side in ("argmin", "argmax"):
            if w[side] is None:
                assert e[side] is None
            else:
                rhs, vr = w[side]
                row_of = {int(vr[r]): r for r in range(1, len(vr))}
                for y in m.variables:
                    val = fixed[y] if y in fixed else (float(rhs[row_of[y.index]]) if y.index in row_of else 0.0)
                    assert _bits(e[side][y.id]) == _bits(val), (what, x.id, side, y.id)
    for c, e in zip(m.constraints, v["constraints"]):
        w = want[c.index]
        assert e["type"] == ("max" if c.isUpperBound else "min")
        assert same(e["slack"]["min"], w["min"]) and same(e["slack"]["max"], w["max"]), (what, e, w)
    t.close()
    return v


@pytest.mark.parametrize("fx", CONTINUOUS, ids=lambda f: f["file"])
def test_fixture_reports_equal_the_oracle(fx):
    if len(fx["model"]["constraints"]) > 100:
        pytest.skip("the oracle takes minutes on every target of the 600-row fixture; its face is checked below")
    if assert_report(strip_timeouts(fx["model"]), fx["file"]) is None:
        pytest.skip("no optimum")


def test_monster_problem_face_and_sampled_report():
    import jslpsolver_b200 as J
    jm = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Monster Problem.json"][0]["model"])
    sol = J.Solve(jm, full=True)
    t = sol._tableau
    t.set_option(3, 1 << 20)
    f, kept, F, vcol_f = assert_face(t, "Monster Problem")
    if f is not None:
        assert_targets(t, f, F, vcol_f, _all_targets(t, kept)[::37], "Monster Problem")
        f.close()
    v = sol.variability(variables=list(jm["variables"])[::40], constraints=list(jm["constraints"])[::40])
    assert v["free"] == len(kept) - 1 and len(v["variables"]) == len(list(jm["variables"])[::40])
    t.close()


def test_seeded_and_known_reports():
    from jslpsolver_b200 import problems
    hand = {"optimize": "profit", "opType": "max",
            "constraints": {"both": {"max": 4}, "capx": {"max": 3}, "capy": {"max": 3}},
            "variables": {"x": {"profit": 1, "both": 1, "capx": 1}, "y": {"profit": 1, "both": 1, "capy": 1}}}
    v = assert_report(hand, "hand example")
    assert v["unique"] is False
    for vid in ("x", "y"):
        assert (v["variables"][vid]["min"], v["variables"][vid]["max"]) == (1.0, 3.0)
    berlin = {"optimize": "capacity", "opType": "max",
              "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
              "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                            "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}
    assert assert_report(berlin, "Berlin Airlift")["unique"] is True
    fixed = {"optimize": "z", "opType": "max", "constraints": {"lo": {"max": -2}, "hi": {"max": 2}, "cap": {"max": 7}},
             "variables": {"x": {"z": 1, "lo": -1, "hi": 1, "cap": 1}, "y": {"z": 2, "cap": 1}, "w": {"z": 2, "cap": 1}}}
    v = assert_report(fixed, "presolve-fixed x")
    assert v["variables"]["x"]["fixed"] and (v["variables"]["y"]["min"], v["variables"]["y"]["max"]) == (0.0, 5.0)
    for seed in range(3):
        v = assert_report(problems.alternative_optima_model(24 + seed, 12 + seed, seed=40 + seed), f"alt seed {seed}")
        assert v["free"] >= 2 and not v["unique"]
    assert assert_report(problems.dense_packing_lp_model(30, 20, seed=2), "dense 30x20") is not None

"""GPU checks of near-optimal variability (DESIGN.md section 2i): jslp_bound_create against the restatement in
near_optimal_oracle.py bit for bit (the shape, every double of B at its logical width with its +0 cost row and
sign-flipped bound row, vrow', vcol', nVars and lastElementIndex) on solved seeded LPs with ping-pong on and off, on the
2001 x 2001 benchmark optimum, at the column-tile edges of k_bound_rows and with +-0, +-P and NaN cost entries; every
target LP on B (status, pivot counts, raw evaluation, column 0, row labels) against the oracle on the shared-memory
batch, on engine 2 and on a tableau beyond shared memory; the parent tableau untouched; and
Solution.variability(gap=...) equal to the restatement's end to end, with sensitivity(), scenarios(), basis() and
variability() unchanged afterwards."""
import math

import numpy as np
import pytest

import near_optimal_oracle as NO
import test_gpu_variability as GV
from conftest import load_bundle
from helpers import strip_timeouts

pytestmark = pytest.mark.gpu
BUNDLE = load_bundle()
P = 1e-8
_bits = GV._bits


def _label(g):
    return NO.fresh_label(g.nVars, g.lastElementIndex)


def assert_bound(g, t, what="", label=None):
    """g.bound(t) against near_optimal_oracle.bound on g's own tableau; returns (bound tab, B, vrow', vcol').  `label`
    is l*, by default that of a freshly uploaded parent (its n_index is nVars)."""
    before = GV._state(g)
    M, vrow, vcol = g.matrix2d().copy(), g.varIndexByRow.copy(), g.varIndexByCol.copy()
    label = _label(g) if label is None else label
    B, vrow_b, vcol_b = NO.bound(M, vrow, vcol, t, label)
    b = g.bound(t)
    assert GV._state(g) == before, f"{what}: the parent tableau changed"
    assert (b.height, b.width) == B.shape == (g.height + 1, g.width), what
    Bg = b.matrix2d()
    assert np.array_equal(_bits(Bg), _bits(B)), (what, "B bits", int((_bits(Bg) != _bits(B)).sum()))
    assert not np.signbit(Bg[0]).any() and (Bg[0] == 0).all(), (what, "row 0 is +0")
    assert np.array_equal(b.varIndexByRow[1:], vrow_b[1:]) and np.array_equal(b.varIndexByCol[1:], vcol_b[1:]), what
    assert (b.nVars, b.lastElementIndex) == (g.nVars + 1, label + 1), what
    return b, B, vrow_b, vcol_b


def assert_targets(b, B, vrow_b, vcol_b, targets, what=""):
    """The (label, sense) targets as one scenario batch on the bound tableau against the oracle's rule 2."""
    from oracle import variability as OV
    out = b.scenario_batch([(1, lab, float(-s)) for lab, s in targets], list(range(len(targets) + 1)), check_cycles=True)
    seen = set()
    for k, (lab, s) in enumerate(targets):
        status, ev, p1, p2, rhs, vr = OV.target(B, vrow_b, vcol_b, P, lab, s)
        got = (int(out["status"][k]), int(out["p1"][k]), int(out["p2"][k]))
        assert got == (status, p1, p2), (what, k, lab, s, got, (status, p1, p2))
        if status == 0:
            assert _bits(out["eval_raw"][k]) == _bits(ev), (what, k, "eval_raw", out["eval_raw"][k], ev)
        assert np.array_equal(_bits(out["rhs"][k]), _bits(rhs)), (what, k, "column 0 bits")
        assert np.array_equal(out["vrow"][k][1:], vr[1:]), (what, k, "row labels")
        seen.add(status)
    return seen, out


def _all_targets(g):
    """Rule 3 for every label of the tableau: two LPs per basic label, one per non-basic label."""
    t = []
    for lab in g.varIndexByRow[1:]:
        t += [(int(lab), -1), (int(lab), 1)]
    return t + [(int(lab), 1) for lab in g.varIndexByCol[1:]]


def _allowance(g, gap):
    return NO.allowance(gap, 0.0, g.cost_row()[0])


# ---------------------------------------------------------------- the bound tableau
@pytest.mark.parametrize("case", ["alt 40x24", "alt 150x120", "dense 150x120", "alt 550x600"])
def test_bound_of_seeded_optima(case):
    from jslpsolver_b200 import _lib, problems
    it = {"alt 40x24": lambda: GV._alt(40, 24, 3), "alt 150x120": lambda: GV._alt(150, 120, 12345),
          "dense 150x120": lambda: problems.dense_packing_lp_tableau(150, 120, 5),
          "alt 550x600": lambda: GV._alt(550, 600, 7)}[case]()
    for pingpong in (1, 0):  # the optimum can end in either buffer of the pair: the bound row reads whichever is current
        g = GV._solved(it, 0, {_lib.OPT_PINGPONG: pingpong})
        for t in (_allowance(g, 0.01), 1e-300, 0.0):
            b, _, _, _ = assert_bound(g, t, f"{case} pingpong {pingpong} t {t}")
            b.close()
        g.close()


def test_config3_optimum():
    """The 2001 x 2001 benchmark LP: its bound tableau, and a few targets on the single-tableau path B takes."""
    from jslpsolver_b200 import problems
    g = GV._solved(problems.dense_packing_lp_tableau(2000, 2000, 12345))
    b, B, vrow_b, vcol_b = assert_bound(g, _allowance(g, 0.01), "config 3")
    tg = _all_targets(g)
    basic = [x for x in tg if x[1] == -1]
    seen, _ = assert_targets(b, B, vrow_b, vcol_b, basic[:2] + [tg[-1]], "config 3")
    assert 0 in seen
    b.close()
    g.close()


def _crafted(H, W, seed):
    """An H x W tableau (not solved: the bound reads any tableau) with signed zeros, +-P, NaN and infinities in its
    cost row and body."""
    M, vrow, vcol = GV._crafted(H, W, set(), seed)
    special = [0.0, -0.0, P, -P, math.nan, -math.nan, 1e-300, -math.inf, math.inf, 5.5]
    M[0, 1:] = [special[(c + seed) % len(special)] for c in range(1, W)]
    M[0, 0] = -123.25
    if H > 2:
        M[1, 1], M[H - 1, W - 1] = -0.0, math.nan
    return M, vrow, vcol


@pytest.mark.parametrize("W", [2, 15, 16, 17, 255, 256, 257, 511, 512, 513, 1025])
def test_column_tile_edges(W):
    """Tiles of 256 columns of the stride in k_bound_rows (stride = ceil16(W): 16, 16, 32, 256, 256, 272, ...), with B's
    height H + 1 on both sides of 64 and of the 32 / 256 row counts the other kernels block by."""
    for H in (1, 2, 31, 32, 63, 64, 255, 256):
        M, vrow, vcol = _crafted(H, W, seed=W + H)
        g = GV._upload(M, vrow, vcol)
        b, B, _, _ = assert_bound(g, 7.75, f"W {W} H {H}")
        assert _bits(B[H, 1:]).tolist() == (_bits(M[0, 1:]) ^ NO.SIGN_BIT).tolist()
        b.close()
        g.close()


def test_removed_variable_keeps_the_wider_stride():
    """removeVariable leaves the parent's stride wider than ceil16(W): rows 1..H-1 are then copied at the logical
    width, row by row."""
    M, vrow, vcol = _crafted(9, 33, seed=4)
    g = GV._upload(M, vrow, vcol)
    g.removeVariable(int(vcol[20]))
    assert g.width == 32
    b, _, _, _ = assert_bound(g, 1.5, "removed variable", label=max(9 + 33 - 2, g.lastElementIndex))
    b.close()
    g.close()


def test_refusals():
    from jslpsolver_b200._lib import JslpError
    from jslpsolver_b200.tableau import GpuTableau
    M, vrow, vcol = _crafted(4, 6, seed=4)
    g = GV._upload(M, vrow, vcol)
    for t in (-1.0, math.nan, math.inf, -0.5e-300):
        with pytest.raises(JslpError, match="allowance must be finite"):
            g.bound(t)
    g.close()
    g = GpuTableau(P)
    g.upload(M, vrow, vcol, optionalCosts=np.ones((1, 6)))
    with pytest.raises(JslpError, match="optional objectives"):
        g.bound(1.0)
    g.close()


# ---------------------------------------------------------------- the target LPs on the bound tableau
@pytest.mark.parametrize("engine", [0, 2])
def test_targets_match_the_oracle(engine):
    """Every target of two seeded optima: engine 0 runs them one CTA each in shared memory, engine 2 one after
    another on the single-tableau path."""
    seen = set()
    for n, m, seed, kw, gap in ((30, 16, 3, {}, 0.01), (60, 40, 11, {"dup": 6, "par": 5}, 0.002)):
        g = GV._solved(GV._alt(n, m, seed, **kw), engine)
        b, B, vrow_b, vcol_b = assert_bound(g, _allowance(g, gap), f"alt {n}x{m}")
        before = GV._state(g)
        s, out = assert_targets(b, B, vrow_b, vcol_b, _all_targets(g), f"alt {n}x{m} engine {engine}")
        seen |= s
        assert (out["p1"] + out["p2"]).max() > 0, "some target pivots"
        assert GV._state(g) == before
        b.close()
        g.close()
    assert 0 in seen


def test_bound_beyond_shared_memory():
    """A 601 x 551 optimum: B is 602 x 551, beyond shared memory, so its targets run on the single-tableau path."""
    from jslpsolver_b200 import problems
    g = GV._solved(problems.dense_packing_lp_tableau(550, 600, 11))
    b, B, vrow_b, vcol_b = assert_bound(g, _allowance(g, 0.005), "601x551")
    tg = _all_targets(g)
    s, out = assert_targets(b, B, vrow_b, vcol_b, tg[::211], "601x551")
    assert 0 in s and (out["p1"] + out["p2"]).max() > 0
    b.close()
    g.close()


# ---------------------------------------------------------------- Solution.variability(gap=...) end to end
def assert_report(jm, what, gap=0.0, absolute_gap=0.0):
    import jslpsolver_b200 as J
    sol = J.Solve(jm, full=True)
    if not (sol.feasible and sol.bounded):
        return None
    t, m = sol._tableau, sol._tableau.model
    rep, scen, basis, exact = sol.sensitivity(), sol.scenarios([{}]), sol.basis(), sol.variability(points=True)
    t.set_option(3, 1 << 20)  # JSLP_OPT_PIVOT_LOG_CAP
    before = GV._state(t)
    v = sol.variability(points=True, gap=gap, absolute_gap=absolute_gap)
    assert GV._state(t) == before, f"{what}: the caller's tableau changed"
    assert sol.sensitivity() == rep and sol.scenarios([{}]) == scen and sol.basis() == basis
    assert sol.variability(points=True) == exact and sol.variability(points=True, gap=0.0) == exact
    assert not any("Cycle" in str(x) for x in m.messages)
    t._cache.clear()
    M, vrow, vcol = t.matrix2d().copy(), t.varIndexByRow.copy(), t.varIndexByCol.copy()
    allowance = NO.allowance(gap, absolute_gap, M[0, 0])
    assert v["allowance"] == allowance > 0
    fixed = m.presolveResult.fixedVariables if m.presolveResult is not None else {}
    labels = [x.index for x in m.variables if x not in fixed] + [c.index for c in m.constraints]
    want, free, lps, _ = NO.ranges(M, vrow, vcol, t.precision, labels, allowance, _label(t))
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
                continue
            rhs, vr = w[side]
            row_of = {int(vr[r]): r for r in range(1, len(vr))}
            for y in m.variables:
                val = fixed[y] if y in fixed else (float(rhs[row_of[y.index]]) if y.index in row_of else 0.0)
                assert _bits(e[side][y.id]) == _bits(val), (what, x.id, side, y.id)
    for c, e in zip(m.constraints, v["constraints"]):
        w = want[c.index]
        assert same(e["slack"]["min"], w["min"]) and same(e["slack"]["max"], w["max"]), (what, e, w)
    t.close()
    return v


@pytest.mark.parametrize("fx", GV.CONTINUOUS, ids=lambda f: f["file"])
def test_fixture_reports_equal_the_oracle(fx):
    if len(fx["model"]["constraints"]) > 100:
        pytest.skip("the oracle would run an LP per structural variable of the 600-row fixture; see the 601 x 551 case")
    if assert_report(strip_timeouts(fx["model"]), fx["file"], gap=0.01) is None:
        pytest.skip("no optimum")


def test_seeded_and_known_reports():
    from jslpsolver_b200 import problems
    hand = {"optimize": "profit", "opType": "max",
            "constraints": {"both": {"max": 4}, "capx": {"max": 3}, "capy": {"max": 3}},
            "variables": {"x": {"profit": 1, "both": 1, "capx": 1}, "y": {"profit": 1, "both": 1, "capy": 1}}}
    v = assert_report(hand, "hand example", absolute_gap=1.0)
    for vid in ("x", "y"):  # x + y >= 3, x, y <= 3
        assert (v["variables"][vid]["min"], v["variables"][vid]["max"]) == (0.0, 3.0)
    berlin = {"optimize": "capacity", "opType": "max",
              "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
              "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                            "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}
    v = assert_report(berlin, "Berlin Airlift", gap=0.05)
    assert abs(v["allowance"] - 0.05 * 1080000.0) < 1e-6 and not v["unique"]
    fixed = {"optimize": "z", "opType": "max", "constraints": {"lo": {"max": -2}, "hi": {"max": 2}, "cap": {"max": 7}},
             "variables": {"x": {"z": 1, "lo": -1, "hi": 1, "cap": 1}, "y": {"z": 2, "cap": 1}, "w": {"z": 2, "cap": 1}}}
    v = assert_report(fixed, "presolve-fixed x", absolute_gap=3.0)
    assert v["variables"]["x"]["fixed"] and (v["variables"]["y"]["min"], v["variables"]["y"]["max"]) == (0.0, 5.0)
    for seed in range(3):
        assert_report(problems.alternative_optima_model(24 + seed, 12 + seed, seed=40 + seed), f"alt seed {seed}",
                      gap=0.02)
    assert assert_report(problems.dense_packing_lp_model(30, 20, seed=2), "dense 30x20", gap=0.001) is not None
    checked = 0
    for k in range(30):
        checked += assert_report(problems.mixed_lp_model(12, 9, seed=900 + k), f"mixed {k}", absolute_gap=2.0) is not None
        if checked >= 2:
            return
    pytest.fail(f"only {checked} seeded mixed LPs had an optimum")

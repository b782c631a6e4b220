"""GPU checks of lexicographic objectives (DESIGN.md section 2j): jslp_lex_next against the restatement in
lexicographic_oracle.py bit for bit (every double of the next level's tableau at its logical width, vrow', vcol', the
kept columns, nVars and lastElementIndex) for the face and the bound kind, on seeded optima with ping-pong on and off,
on the 2001 x 2001 benchmark optimum and on a parent left wider by removeVariable; the pricing at k_price_objective's
column-tile and row-block edges with +-0 coefficients, empty blocks and +-0, +-P, NaN and +-inf costs; row 0 against
jslp_frontier's R2 on the same parent; every level of face, bound and mixed chains (status, no phase-1 pivot, phase-2
pivots, M[0,0], column 0, labels) after solves on engines 0, 1, 2 and 4; the parent left as it was; and
Lexicographic() equal to the restatement end to end."""
import math

import numpy as np
import pytest

import lexicographic_oracle as LO
import near_optimal_oracle as NO
import test_gpu_variability as GV

pytestmark = pytest.mark.gpu
P = 1e-8
ENGINES = (0, 1, 2, 4)
_bits = GV._bits


def _same(a, b):
    """Bit for bit, except that any NaN matches any NaN (a product with a NaN or an infinite cost need not keep the
    payload NumPy keeps)."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all((_bits(a) == _bits(b)) | (np.isnan(a) & np.isnan(b))))


def assert_child(g, cost, t, what=""):
    """g.lex_next(cost, t) against lexicographic_oracle.child on g's own tableau; returns (next, T, vrow', vcol')."""
    before = GV._state(g)
    M, vrow, vcol = g.matrix2d().copy(), g.varIndexByRow.copy(), g.varIndexByCol.copy()
    label = NO.fresh_label(g.nVars, g.lastElementIndex)
    T, vr, vc, kept = LO.child(M, vrow, vcol, P, cost, t, label)
    nxt, got = g.lex_next(cost, t)
    assert GV._state(g) == before, f"{what}: the parent tableau changed"
    assert np.array_equal(got, kept), (what, "kept columns", got[:8], kept[:8], len(got), len(kept))
    if T is None:
        assert nxt is None, what
        return None, None, None, None
    assert (nxt.height, nxt.width) == T.shape, (what, (nxt.height, nxt.width), T.shape)
    Tg = nxt.matrix2d()
    assert _same(Tg, T), (what, "bits", int((~((_bits(Tg) == _bits(T)) | (np.isnan(Tg) & np.isnan(T)))).sum()))
    assert np.array_equal(nxt.varIndexByRow[1:], vr[1:]) and np.array_equal(nxt.varIndexByCol[1:], vc[1:]), what
    want = (g.nVars, g.lastElementIndex) if t == 0.0 else (g.nVars + 1, label + 1)
    assert (nxt.nVars, nxt.lastElementIndex) == want, (what, nxt.nVars, nxt.lastElementIndex, want)
    return nxt, T, vr, vc


def _cost(g, seed, zeros=0.3):
    """A seeded objective by label: sigma * U{1..20} at a share of the labels, 0 elsewhere."""
    rng = np.random.default_rng(seed)
    c = rng.integers(1, 21, size=g.nVars).astype(np.float64) * rng.choice([-1.0, 1.0])
    c[rng.random(g.nVars) < zeros] = 0.0
    return c


# ---------------------------------------------------------------- the next level's tableau
@pytest.mark.parametrize("case", ["alt 40x24", "alt 150x120", "dense 150x120", "alt 550x600"])
def test_child_of_seeded_optima(case):
    from jslpsolver_b200 import _lib, problems
    it = {"alt 40x24": lambda: GV._alt(40, 24, 3), "alt 150x120": lambda: GV._alt(150, 120, 12345),
          "dense 150x120": lambda: problems.dense_packing_lp_tableau(150, 120, 5),
          "alt 550x600": lambda: GV._alt(550, 600, 7)}[case]()
    for pingpong in (1, 0):  # the optimum can end in either buffer of the pair: the child reads whichever is current
        g = GV._solved(it, 0, {_lib.OPT_PINGPONG: pingpong})
        for seed, t in ((1, 0.0), (2, NO.allowance(0.01, 0.0, g.cost_row()[0])), (3, 1e-300)):
            nxt, _, _, _ = assert_child(g, _cost(g, seed), t, f"{case} pingpong {pingpong} t {t}")
            if nxt is not None:
                nxt.close()
        g.close()


def test_config3_optimum():
    """The 2001 x 2001 benchmark optimum: the bound kind at 1 % and the face kind."""
    from jslpsolver_b200 import problems
    g = GV._solved(problems.dense_packing_lp_tableau(2000, 2000, 12345))
    cost = _cost(g, 7)
    for t in (NO.allowance(0.01, 0.0, g.cost_row()[0]), 0.0):
        nxt, _, _, _ = assert_child(g, cost, t, f"config 3 t {t}")
        if nxt is not None:
            nxt.close()
    g.close()


def test_removed_variable_keeps_the_wider_stride():
    """removeVariable leaves the parent's stride wider than ceil16(W): both kinds read it at its logical width."""
    M, vrow, vcol = GV._crafted(9, 33, {3, 7, 20, 31}, seed=4)
    g = GV._upload(M, vrow, vcol)
    g.removeVariable(int(vcol[20]))
    assert g.width == 32
    for t in (0.0, 1.5):
        nxt, _, _, _ = assert_child(g, _cost(g, 5), t, f"removed variable t {t}")
        nxt.close()
    g.close()


SPECIAL = [0.0, -0.0, P, -P, np.nextafter(P, 1.0), np.nextafter(-P, -1.0), math.nan, math.inf, -math.inf, 3.0, -2.5]


@pytest.mark.parametrize("W", [127, 128, 129, 255, 256, 257])
def test_pricing_edges(W):
    """Column tiles of 128 outputs and row blocks of 64 of k_price_objective (H - 1 = 63..65 and 127..129), with +-0
    coefficients in the body, a row block whose basic labels all cost 0, and costs of +-0, +-P, one ulp beyond P, NaN
    and +-inf; the face kind through the kept-column map and the bound kind over every column."""
    for H in (64, 65, 66, 128, 129, 130):
        keep = set(range(1, W, 3))
        M, vrow, vcol = GV._crafted(H, W, keep, seed=W * 1000 + H)
        M[1:, 5] = -0.0
        M[2, 1:] = 0.0
        g = GV._upload(M, vrow, vcol)
        cost = np.array([SPECIAL[(lab * 7 + H) % len(SPECIAL)] for lab in range(g.nVars)])
        cost[[int(x) for x in vrow[1:min(H, 65)]]] = 0.0  # the first row block has no non-zero coefficient
        if H > 66:
            cost[int(vrow[70])] = -0.0
        for t in (0.0, 2.0):
            nxt, _, _, _ = assert_child(g, cost, t, f"W {W} H {H} t {t}")
            nxt.close()
        g.close()


def test_refusals():
    from jslpsolver_b200._lib import JslpError
    from jslpsolver_b200.tableau import GpuTableau
    M, vrow, vcol = GV._crafted(4, 6, {1, 2}, seed=4)
    g = GV._upload(M, vrow, vcol)
    for t in (-1.0, math.nan, math.inf, -0.5e-300):
        with pytest.raises(JslpError, match="allowance must be finite"):
            g.lex_next(np.zeros(g.nVars), t)
    with pytest.raises(ValueError, match="entries"):
        g.lex_next(np.zeros(g.nVars + 1), 0.0)
    g.close()
    g = GpuTableau(P)
    g.upload(M, vrow, vcol, optionalCosts=np.ones((1, 6)))
    with pytest.raises(JslpError, match="optional objectives"):
        g.lex_next(np.zeros(g.nVars), 1.0)
    g.close()


def test_row_zero_is_the_frontier_pricing():
    """Row 0 of the next level is jslp_frontier's R2 on the same parent, at the kept columns."""
    from jslpsolver_b200 import problems
    g = GV._solved(problems.dense_packing_lp_tableau(150, 120, 9))
    for seed in (11, 12):
        cost = _cost(g, seed)
        r2 = g.frontier_path(cost, 4 * (g.height + g.width))["r2"]
        for t in (0.0, 3.0):
            nxt, kept = g.lex_next(cost, t)
            if nxt is None:
                continue
            assert np.array_equal(_bits(nxt.matrix2d()[0]), _bits(r2[kept])), (seed, t)
            nxt.close()
    g.close()


# ---------------------------------------------------------------- every level
def _levels_on_device(jm, gap, engine, what):
    """The chain of jm level by level on the device, each level against the restatement from the device's own parent;
    returns the kinds run."""
    import jslpsolver_b200 as J
    from jslpsolver_b200 import frontier as HF
    s = J.Solver()
    s.engine = engine
    keys = list(jm["optimize"])
    senses = {k: jm["optimize"][k] for k in keys}
    working = dict(jm, optimize=keys[0], opType=senses[keys[0]])
    inst = s._instance(working, None)
    assert inst.solve().feasible
    cur, kinds = inst.tableau, []
    for k in range(1, len(keys)):
        cur._cache.clear()
        z = -(1.0 if senses[keys[k - 1]] == "max" else -1.0) * float(cur.cost_row()[0])
        g = gap[k - 1] if isinstance(gap, (list, tuple)) else gap
        t = g * abs(z)
        cost = np.array(HF.cost_row(inst, working, keys[k], senses[keys[k]], cur.nVars))
        nxt, T, vr, vc = assert_child(cur, cost, t, f"{what} level {k + 1}")
        if cur is not inst.tableau:
            cur.close()
        cur = nxt
        if cur is None:
            kinds.append(None)
            break
        kinds.append("face" if t == 0.0 else "bound")
        status, p1, p2, Mf, vrf, _ = LO.solve(T, vr, vc, P)
        cur.simplex(check_cycles=True)
        st = cur.lastStatus
        got = 3 if st.cycled else 1 if not cur.feasible else 2 if not cur.bounded else 0
        assert (got, st.phase1_pivots, st.phase2_pivots) == (status, 0, p2) and p1 == 0, \
            (what, k, (got, st.phase1_pivots, st.phase2_pivots), (status, p1, p2))
        cur._cache.clear()
        Mg = cur.matrix2d()
        assert _bits(Mg[0, 0]) == _bits(Mf[0, 0]) and np.array_equal(_bits(Mg[:, 0]), _bits(Mf[:, 0])), (what, k)
        assert np.array_equal(cur.varIndexByRow[1:], vrf[1:]), (what, k)
        if status != 0:
            break
    if cur is not None and cur is not inst.tableau:
        cur.close()
    return kinds


@pytest.mark.parametrize("engine", ENGINES)
def test_every_level_matches_the_restatement(engine):
    from jslpsolver_b200 import problems
    kinds = set()
    for n, m, levels, seed in ((30, 16, 3, 1), (60, 40, 5, 2)):
        jm = problems.alternative_optima_multi_model(n, m, levels, seed=seed)
        for gap in (0.0, 0.01, [0.0, 0.01, 0.0, 0.002]):
            kinds |= set(_levels_on_device(jm, gap, engine, f"alt {n}x{m} gap {gap} engine {engine}"))
    kinds |= set(_levels_on_device(problems.dense_packing_multi_model(121, 151, 3, seed=3), 0.01, engine,
                                   f"dense 121x151 engine {engine}"))
    assert {"face", "bound"} <= kinds, kinds


# ---------------------------------------------------------------- Lexicographic() end to end
def test_lexicographic_equals_the_restatement():
    import jslpsolver_b200 as J
    from jslpsolver_b200 import problems
    ray = {"optimize": {"a": "max", "b": "max"}, "constraints": {"gap": {"max": 2}, "cap": {"max": 5}},
           "variables": {"x": {"a": 1, "gap": 1, "cap": 1}, "y": {"b": 1, "gap": -1}}}
    berlin = {"optimize": {"capacity": "max", "cost": "min", "plane": "max"},
              "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
              "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                            "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}
    fixed = {"optimize": {"z": "max", "w2": "min"},
             "constraints": {"lo": {"max": -2}, "hi": {"max": 2}, "cap": {"max": 7}},
             "variables": {"x": {"z": 1, "w2": 5, "lo": -1, "hi": 1, "cap": 1}, "y": {"z": 2, "w2": 1, "cap": 1},
                           "w": {"z": 2, "w2": 3, "cap": 1}}}
    cases = [(problems.alternative_optima_multi_model(24, 12, 3, seed=1), 0.0, 0.0),
             (problems.alternative_optima_multi_model(24, 12, 5, seed=2), 0.01, 0.0),
             (problems.alternative_optima_multi_model(40, 20, 4, seed=3), {"objective": 0.01}, {"obj2": 3.0}),
             (problems.dense_packing_multi_model(60, 40, 3, seed=4), 0.005, 0.0),
             (berlin, 0.0, 0.0), (ray, 0.0, 1.0), (fixed, 0.0, 3.0),
             (dict(problems.planted_infeasible_model(8, 6, 2, seed=4), optimize={"objective": "max", "b": "max"}),
              0.0, 0.0)]
    stops = set()
    for jm, gap, absolute_gap in cases:
        want, _ = LO.chain(jm, gap, absolute_gap)
        got = J.Lexicographic(jm, gap=gap, absolute_gap=absolute_gap)
        assert got == want, (jm.get("name"), got, want)
        stops.add(got["stop"])
    assert {"reached", "unbounded", None} <= stops

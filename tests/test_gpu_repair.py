"""GPU checks of Repair() (DESIGN.md section 2k): jslp_elastic_create against the restatement in repair_oracle.py bit
for bit (every double of E at its logical width, vrow', vcol', nVars, lastElementIndex and the crash count) at
ELASTIC_TILE_ROWS - 1, exactly, + 1 and twice as many crashed rows, at W + k = 255, 256 and 257, with right-hand sides
at exactly -P and one ulp below, signed zeros and non-unit weights, on a parent left wider by removeVariable and on a
2001-row infeasible_packing_model; the parent left as it was; both stages (status, phase-1 / phase-2 pivots, the
pivot sequence, every bit of the final tableau and its labels) against the oracle on engines 0, 1, 2 and 4; the entry
point's refusals; and Repair() equal to the restatement end to end."""
import math

import numpy as np
import pytest

import repair_oracle as RO
import test_gpu_variability as GV
from oracle import ref_model

pytestmark = pytest.mark.gpu
P = 1e-8
ENGINES = (0, 1, 2, 4)
_bits = GV._bits
BERLIN = {"optimize": "capacity", "opType": "max",
          "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
          "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                        "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}
BROKEN = dict(BERLIN, constraints=dict(BERLIN["constraints"], brit={"min": 13}))


def _same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all(_bits(a) == _bits(b)))


def assert_elastic(g, rows, w, what=""):
    """g.elastic(rows, w) against repair_oracle.elastic on g's own tableau; returns (E tab, E, vrow', vcol')."""
    before = GV._state(g)
    M, vrow, vcol = g.matrix2d().copy(), g.varIndexByRow.copy(), g.varIndexByCol.copy()
    label = max(g.nVars, g.lastElementIndex)
    E, vr, vc, crashed = RO.elastic(M, vrow, vcol, P, rows, w, label)
    e, n = g.elastic(rows, w)
    assert GV._state(g) == before, f"{what}: the parent tableau changed"
    assert n == len(crashed), (what, n, len(crashed))
    assert (e.height, e.width) == E.shape, (what, (e.height, e.width), E.shape)
    Eg = e.matrix2d()
    assert _same(Eg, E), (what, "bits", np.argwhere(_bits(Eg) != _bits(E))[:8])
    assert np.array_equal(e.varIndexByRow[1:], vr[1:]) and np.array_equal(e.varIndexByCol[1:], vc[1:]), what
    assert (e.nVars, e.lastElementIndex) == (g.nVars + len(rows), label + len(rows)), (what, e.nVars)
    return e, E, vr, vc


def _crafted(H, W, n_neg, seed, zeros=True):
    """A dense H x W tableau with n_neg seeded rows below -P in column 0, the others above, and signed zeros."""
    rng = np.random.default_rng(seed)
    M = rng.integers(-20, 21, size=(H, W)).astype(np.float64) / 4.0
    if zeros:
        M[rng.random((H, W)) < 0.1] = -0.0
    M[0] = rng.integers(-5, 6, size=W)
    neg = rng.permutation(np.arange(1, H))[:n_neg]
    M[1:, 0] = rng.uniform(1.0, 9.0, H - 1)
    M[neg, 0] = -rng.uniform(1.0, 9.0, len(neg))
    vrow = np.arange(-1, H - 1, dtype=np.int32)
    vcol = np.concatenate([[-1], np.arange(H - 1, H + W - 2)]).astype(np.int32)
    return M, vrow, vcol


# ---------------------------------------------------------------- the elastic tableau
@pytest.mark.parametrize("crashed", [RO.ELASTIC_TILE_ROWS - 1, RO.ELASTIC_TILE_ROWS, RO.ELASTIC_TILE_ROWS + 1,
                                     2 * RO.ELASTIC_TILE_ROWS])
def test_crash_counts_at_the_tile_edges(crashed):
    H = 2 * RO.ELASTIC_TILE_ROWS + 6
    M, vrow, vcol = _crafted(H, 13, crashed, seed=crashed)
    g = GV._upload(M, vrow, vcol)
    rng = np.random.default_rng(crashed)
    rows = list(range(1, H))
    w = list(rng.uniform(0.1, 7.0, len(rows)))
    e, E, _, _ = assert_elastic(g, rows, w, f"{crashed} crashed")
    e.simplex(check_cycles=True)
    assert e.lastStatus.phase1_pivots == 0
    e.close()
    g.close()


@pytest.mark.parametrize("width", [255, 256, 257])
def test_elastic_width_at_the_column_tile_edges(width):
    """W + k = 255, 256, 257 with a subset of the rows relaxable."""
    H = 40
    k = 30
    M, vrow, vcol = _crafted(H, width - k, 12, seed=width)
    g = GV._upload(M, vrow, vcol)
    rows = sorted(np.random.default_rng(width).choice(np.arange(1, H), size=k, replace=False).tolist())
    w = [1.0 + 0.5 * (j % 3) for j in range(k)]
    e, _, _, _ = assert_elastic(g, rows, w, f"W + k = {width}")
    assert e.width == width
    e.close()
    g.close()


def test_thresholds_signed_zeros_and_weights():
    M, vrow, vcol = _crafted(12, 9, 5, seed=3)
    M[2, 0], M[3, 0], M[4, 0], M[5, 0] = -P, -np.nextafter(P, 1.0), -0.0, 0.0
    M[3, 1:4] = [0.0, -0.0, math.inf]
    g = GV._upload(M, vrow, vcol)
    rows = list(range(1, 12))
    w = [0.1, 0.3, 1.0 / 3.0, 7.0, 1e-300, 1e300, 2.5, 0.7, 3.0, 11.0, 0.2]
    e, E, vr, _ = assert_elastic(g, rows, w, "thresholds")
    assert vr[2] == vrow[2] and vr[3] != vrow[3] and vr[4] == vrow[4] and vr[5] == vrow[5]
    assert np.signbit(E[3, 1]) and not np.signbit(E[3, 2]) and E[3, 3] == -math.inf
    e.close()
    # a subset, rows given by one weight each
    e, _, _, _ = assert_elastic(g, [1, 3, 8], [2.0, 0.25, 9.0], "subset")
    e.close()
    e, _, _, _ = assert_elastic(g, [], [], "no row")
    e.close()
    g.close()


def test_removed_variable_keeps_the_wider_stride():
    M, vrow, vcol = _crafted(20, 33, 7, seed=4)
    g = GV._upload(M, vrow, vcol)
    g.removeVariable(int(vcol[20]))
    assert g.width == 32
    e, _, _, _ = assert_elastic(g, list(range(1, 20)), [1.0] * 19, "removed variable")
    e.close()
    g.close()


def test_2001_row_packing_model():
    from jslpsolver_b200 import problems
    A, b, c, lower = problems.infeasible_packing_arrays(2000, 2000, 600, seed=1)
    it = problems.lp_tableau(A, b, c, lower)
    g = GV._upload(it.matrix, it.varIndexByRow, it.varIndexByCol)
    rows = list(range(1, 2001))
    e, _, _, _ = assert_elastic(g, rows, [1.0 + (r % 7) for r in rows], "2001 rows")
    assert e.width == 4001
    e.close()
    g.close()


def test_refusals():
    from jslpsolver_b200._lib import JslpError
    from jslpsolver_b200.tableau import GpuTableau
    M, vrow, vcol = _crafted(6, 5, 2, seed=9)
    g = GV._upload(M, vrow, vcol)
    for rows, w, match in (([2, 1], [1.0, 1.0], "increasing"), ([0], [1.0], "within"), ([6], [1.0], "within"),
                           ([1], [0.0], "finite and > 0"), ([1], [-1.0], "finite and > 0"),
                           ([1], [math.nan], "finite and > 0"), ([1], [math.inf], "finite and > 0")):
        with pytest.raises(JslpError, match=match):
            g.elastic(rows, w)
    g.simplex()  # a pivoted tab no longer has every row's own slack basic
    moved = [r for r in range(1, 6) if g.varIndexByRow[r] != vrow[r]]
    if moved:
        with pytest.raises(JslpError, match="its own slack"):
            g.elastic(moved[:1], [1.0])
    g.close()
    g = GpuTableau(P)
    g.upload(M, vrow, vcol, optionalCosts=np.ones((1, 5)))
    with pytest.raises(JslpError, match="optional objectives"):
        g.elastic([1], [1.0])
    g.close()


# ---------------------------------------------------------------- both stages against the oracle
def _oracle_log(T, vrow, vcol):
    """(row, column) of every pivot the oracle's simplex makes on T with the cycle check on."""
    present = np.array(sorted([int(v) for v in vrow[1:]] + [int(v) for v in vcol[1:]]), dtype=np.int32)
    rank = {int(v): k for k, v in enumerate(present)}
    rename = lambda a: np.array([-1] + [rank[int(v)] for v in a[1:]], dtype=np.int32)  # noqa: E731
    tab = ref_model.OracleTableau(T, rename(vrow), rename(vcol), precision=P,
                                  unrestricted=np.zeros(len(present), dtype=np.uint8), check_cycles=True,
                                  fast_cycles=True, is_min=True, pivot_log=1 << 20)
    tab.simplex()
    return np.asarray(tab.pivot_log())[:, :2]


def _check_stage(tab, T, vr, vc, want, what):
    status, p1, p2, Mx, vrow_f, vcol_f = want
    st = tab.lastStatus
    assert (int(st.phase1_pivots), int(st.phase2_pivots)) == (p1, p2), (what, st.phase1_pivots, st.phase2_pivots, p1, p2)
    assert np.array_equal(tab.pivot_log()[:, :2], _oracle_log(T, vr, vc)), (what, "pivot sequence")
    assert _same(tab.matrix2d(), Mx), (what, "final bits")
    assert np.array_equal(tab.varIndexByRow[1:], vrow_f[1:]) and np.array_equal(tab.varIndexByCol[1:], vcol_f[1:])


@pytest.mark.parametrize("engine", ENGINES)
def test_both_stages_match_the_oracle(engine):
    from jslpsolver_b200 import _lib, problems
    from jslpsolver_b200.repair import objective_row
    from jslpsolver_b200.model import Model
    cases = [(BROKEN, 0.0), (problems.infeasible_packing_model(30, 40, 9, seed=2), 0.0),
             (problems.infeasible_packing_model(30, 40, 9, seed=3), 0.02),
             (problems.planted_infeasible_model(40, 30, 4, seed=5), 0.5)]
    for jm, gap in cases:
        res, det = RO.repair(jm, gap=gap)
        it = Model().loadJson(jm).initial_tableau()
        g = GV._upload(it.matrix, it.varIndexByRow, it.varIndexByCol, engine)
        e, n = g.elastic(det["rows"], det["weights"])
        e.set_option(_lib.OPT_PIVOT_LOG_CAP, 1 << 20)
        assert n == len(det["crashed"])
        e.simplex(check_cycles=True)
        _check_stage(e, det["E"], det["vrow_e"], det["vcol_e"], det["s1"], (engine, jm.get("name"), 1))
        assert e.lastStatus.phase1_pivots == 0
        if det["T"] is None:
            e.close()
            g.close()
            continue
        nxt, _ = e.lex_next(objective_row(it, e.nVars), det["t"])
        assert _same(nxt.matrix2d(), det["T"]), (engine, jm.get("name"), "stage 2 start")
        nxt.set_option(_lib.OPT_PIVOT_LOG_CAP, 1 << 20)
        nxt.simplex(check_cycles=True)
        _check_stage(nxt, det["T"], det["vrow_t"], det["vcol_t"], det["s2"], (engine, jm.get("name"), 2))
        for t in (nxt, e, g):
            t.close()


# ---------------------------------------------------------------- Repair() end to end
def test_repair_equals_the_restatement():
    import jslpsolver_b200 as J
    from jslpsolver_b200 import problems
    cases = [(BROKEN, {}), (BROKEN, {"gap": 0.1}), (BROKEN, {"objective": False}), (BERLIN, {}),
             (BROKEN, {"weights": {"plane": 1.0}}),
             ({"optimize": "z", "opType": "max", "constraints": {"need": {"min": 4}, "cap": {"max": 1}},
               "variables": {"x": {"z": 1, "need": 1, "cap": 1}, "y": {"z": 1}}}, {}),
             (problems.infeasible_packing_model(60, 80, 20, seed=7), {"gap": 0.01}),
             (problems.infeasible_packing_model(60, 80, 20, seed=8), {"weights": {f"c{i}": 1.0 + i % 3 for i in range(80)}}),
             (problems.planted_infeasible_model(30, 20, 3, seed=9), {"absolute_gap": 0.5})]
    for jm, kw in cases:
        want, _ = RO.repair(jm, kw.get("weights"), kw.get("objective", True), kw.get("gap", 0.0),
                            kw.get("absolute_gap", 0.0))
        got = J.Repair(jm, **kw)
        assert got == want, (jm.get("name"), kw, got, want)
    out = J.Solver().Repair(BROKEN)
    assert out["violation"] == 13.0 and out["result"] == 1080000.0 and out["values"] == {"brit": 24.0, "yank": 20.0}
    assert not J.Solve(BROKEN)["feasible"]

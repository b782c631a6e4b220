"""GPU checks of Solution.unbounded() (DESIGN.md section 2l): jslp_cone_create against the restatement in
unbounded_oracle.py bit for bit (every double of the cone at its logical width, signed zeros in column 0 and row 0,
the labels, nVars and lastElementIndex) at k_cone_rows' tile edges, on a parent left wider by removeVariable and at
2001 rows; jslp_column against matrix2d() for every column of stop tableaux at width and stride edges;
jslp_column_batch against the oracle set by set (status, eval bits, pivots, final column 0 bits and labels) on the
shared-memory and single-tableau paths, on engines 0, 1, 2 and 4, with random, empty and all-column masks, a log cap
small enough to send sets to the single-tableau path and a Beale-type cone that cycles, with the snapshot and scalar
state unchanged afterwards; and Solution.unbounded() equal to the restatement end to end."""
import numpy as np
import pytest

import test_gpu_variability as GV
import unbounded_oracle as UO
from helpers import strip_timeouts

pytestmark = pytest.mark.gpu
P = 1e-8
ENGINES = (0, 1, 2, 4)
_bits = GV._bits
CODE = {UO.OPTIMAL: 0, UO.UNBOUNDED: 1, UO.CYCLED: 2, UO.INFEASIBLE: 3}
EXAMPLE = {"optimize": "profit", "opType": "max",
           "constraints": {"c": {"max": 4}, "d": {"min": 1}},
           "variables": {"x": {"profit": 1, "c": 1, "d": 1}, "y": {"profit": 2, "c": -1}}}
SPURIOUS = {"optimize": "x", "opType": "max", "constraints": {"c": {"max": 5e-8}}, "variables": {"x": {"x": 1, "c": 10}}}


def _same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all(_bits(a) == _bits(b)))


def _crafted(H, W, seed):
    """A dense H x W tableau with signed zeros in column 0 and row 0 and an identity labelling."""
    rng = np.random.default_rng(seed)
    M = rng.integers(-20, 21, size=(H, W)).astype(np.float64) / 4.0
    M[rng.random((H, W)) < 0.1] = -0.0
    M[1::3, 0] = -0.0
    M[0, 1::4] = -0.0
    vrow = np.arange(-1, H - 1, dtype=np.int32)
    vcol = np.concatenate([[-1], np.arange(H - 1, H + W - 2)]).astype(np.int32)
    return M, vrow, vcol


def assert_cone(g, what=""):
    """g.cone() against unbounded_oracle.cone on g's own tableau; returns (cone tab, K, vrow', vcol')."""
    before = GV._state(g)
    M, vrow, vcol = g.matrix2d().copy(), g.varIndexByRow.copy(), g.varIndexByCol.copy()
    label = max(g.nVars, g.lastElementIndex)
    K, vr, vc = UO.cone(M, vrow, vcol, label)
    k = g.cone()
    assert GV._state(g) == before, f"{what}: the parent tableau changed"
    assert (k.height, k.width) == K.shape, (what, (k.height, k.width), K.shape)
    assert _same(k.matrix2d(), K), (what, np.argwhere(_bits(k.matrix2d()) != _bits(K))[:8])
    assert np.array_equal(k.varIndexByRow[1:], vr[1:]) and np.array_equal(k.varIndexByCol[1:], vc[1:]), what
    assert (k.nVars, k.lastElementIndex) == (g.nVars + 1, label + 1), what
    return k, K, vr, vc


# ---------------------------------------------------------------- the cone tableau
@pytest.mark.parametrize("H,W", [(12, 255), (12, 256), (12, 257), (255, 9), (256, 9), (257, 9)])
def test_cone_at_the_tile_edges(H, W):
    M, vrow, vcol = _crafted(H, W, seed=H + W)
    g = GV._upload(M, vrow, vcol)
    k, _, _, _ = assert_cone(g, f"{H} x {W}")
    assert not np.signbit(k.matrix2d()[:, 0]).any()  # -0 in column 0 becomes +0
    k.close()
    g.close()


def test_cone_of_a_parent_left_wider_by_remove_variable():
    M, vrow, vcol = _crafted(20, 33, seed=4)
    g = GV._upload(M, vrow, vcol)
    g.removeVariable(int(vcol[20]))
    assert g.width == 32
    k, _, _, _ = assert_cone(g, "removed variable")
    k.close()
    g.close()


def test_cone_at_2001_rows():
    from jslpsolver_b200 import problems
    it = problems.dense_packing_lp_tableau(60, 2000, seed=3)
    g = GV._upload(it.matrix, it.varIndexByRow, it.varIndexByCol)
    k, _, _, _ = assert_cone(g, "2001 rows")
    assert k.height == 2002
    k.close()
    g.close()


# ---------------------------------------------------------------- one column of a stop tableau
@pytest.mark.parametrize("n_vars", [15, 16, 17, 31, 32, 33])
def test_column_equals_matrix2d(n_vars):
    from jslpsolver_b200 import problems
    jm = problems.planted_unbounded_model(n_vars, 14, 1, 1, seed=n_vars)
    m = UO.presolved_model(jm)
    it = m.initial_tableau()
    g = GV._upload(it.matrix, it.varIndexByRow, it.varIndexByCol)
    g.simplex(check_cycles=True)
    assert not g.bounded
    full = g.matrix2d()
    for c in range(g.width):
        assert _same(g.column(c), full[:, c]), c
    g.close()


# ---------------------------------------------------------------- column-subset batches
def _masks(W, n, seed):
    rng = np.random.default_rng(seed)
    keep = (rng.random((n, W)) < 0.7).astype(np.uint8)
    keep[0] = 1          # nothing capped
    keep[1, 1:] = 0      # every column capped
    keep[:, 0] = rng.integers(0, 2, n)  # column 0 is kept whatever the mask says
    return keep


def assert_batch(k, K, vr, vc, keep, what=""):
    k.save()
    before = GV._state(k)[:4]  # tableau, labels and pivot log, evaluation, feasible, bounded (not the edit counter)
    res = k.column_batch(keep)
    assert GV._state(k)[:4] == before, f"{what}: the snapshot or the scalar state was not restored"
    for i in range(len(keep)):
        capped = [c for c in range(1, K.shape[1]) if not keep[i, c]]
        status, piv, Mx, vrow_f = UO.solve(K, vr, vc, P, capped)
        got = (int(res["status"][i]), int(res["pivots"][i]))
        assert got == (CODE[status], piv), (what, i, got, (CODE[status], piv))
        if status != UO.CYCLED:
            assert _bits(res["eval_raw"][i]) == _bits(Mx[0, 0]), (what, i)
        assert _same(res["rhs"][i], Mx[:, 0]), (what, i)
        assert np.array_equal(res["vrow"][i][1:], vrow_f[1:]), (what, i)
    return res


def _planted_cone(n_vars, n_cons, seed, engine=0, options=None):
    from jslpsolver_b200 import problems
    m = UO.presolved_model(problems.planted_unbounded_model(n_vars, n_cons, 3, 2, seed))
    it = m.initial_tableau()
    g = GV._upload(it.matrix, it.varIndexByRow, it.varIndexByCol, engine, options)
    k, K, vr, vc = assert_cone(g)
    return g, k, K, vr, vc


@pytest.mark.parametrize("engine", ENGINES)
def test_column_batch_shared_memory_size(engine):
    g, k, K, vr, vc = _planted_cone(40, 30, seed=engine + 1, engine=engine)
    assert_batch(k, K, vr, vc, _masks(K.shape[1], 24, engine), f"engine {engine}")
    k.close()
    g.close()


@pytest.mark.parametrize("engine", (0, 2))
def test_column_batch_beyond_shared_memory(engine):
    g, k, K, vr, vc = _planted_cone(180, 170, seed=7, engine=engine)
    assert K.shape[0] * K.shape[1] * 8 > 232448  # the cone does not fit one CTA's shared memory
    assert_batch(k, K, vr, vc, _masks(K.shape[1], 5, 7), f"HBM engine {engine}")
    k.close()
    g.close()


def test_column_batch_log_cap_overflow_reruns():
    from jslpsolver_b200 import _lib
    g, k, K, vr, vc = _planted_cone(40, 30, seed=11, options={_lib.OPT_NODE_LOG_CAP: 3})
    res = assert_batch(k, K, vr, vc, _masks(K.shape[1], 16, 11), "log cap 3")
    assert (res["pivots"] > 3).any()  # some sets overflowed the in-kernel log and ran again
    k.close()
    g.close()


def _beale_cone():
    rows = [[0.25, -8, -1, 9], [0.5, -12, -0.5, 3], [0, 0, 1, 0]]
    cost = [0.75, -20, 0.5, -6]
    H, W = len(rows) + 1, len(cost) + 1
    M = np.zeros((H, W))
    M[0, 1:] = cost
    M[1:, 1:] = rows
    vrow = np.arange(-1, H - 1, dtype=np.int32)
    vcol = np.concatenate([[-1], np.arange(H - 1, H + W - 2)]).astype(np.int32)
    return M, vrow, vcol


@pytest.mark.parametrize("engine", ENGINES)
def test_column_batch_cycling_cone_is_undecided(engine):
    M, vrow, vcol = _beale_cone()
    g = GV._upload(M, vrow, vcol, engine)
    k, K, vr, vc = assert_cone(g, "Beale")
    assert UO.solve(K, vr, vc, P, [])[0] == UO.CYCLED
    keep = np.ones((3, K.shape[1]), dtype=np.uint8)
    keep[1, 2] = 0
    res = assert_batch(k, K, vr, vc, keep, f"Beale engine {engine}")
    assert res["status"][0] == 2
    k.close()
    g.close()


# ---------------------------------------------------------------- Solution.unbounded() end to end
def _cases():
    from jslpsolver_b200 import problems
    out = [EXAMPLE, SPURIOUS]
    out += [problems.planted_unbounded_model(*p) for p in ((30, 20, 3, 2, 1), (40, 30, 0, 3, 2), (14, 8, 1, 3, 5))]
    return out


@pytest.mark.parametrize("width", [1, 8, None])
def test_unbounded_equals_the_restatement(width):
    import jslpsolver_b200 as J
    for jm in _cases():
        want = UO.unbounded(UO.presolved_model(jm))
        sol = J.Solve(jm, full=True)
        t = sol._tableau
        before = GV._state(t)
        got = sol.unbounded(width=width)
        assert GV._state(t) == before, "the user's tableau changed"
        if width != 1:
            want.pop("lps"), got.pop("lps")
        assert got == want, (jm.get("name"), width)
        if jm.get("name", "").startswith("Planted"):
            assert got["bound"]["variables"] == [v for v in jm["variables"] if v.startswith(("solo", "pairV"))]
    assert J.Solve(SPURIOUS, full=True).unbounded()["confirmed"] is False


def test_unbounded_refusals():
    import jslpsolver_b200 as J
    bounded = {"optimize": "p", "opType": "max", "constraints": {"c": {"max": 4}}, "variables": {"x": {"p": 1, "c": 1}}}
    infeasible = dict(bounded, constraints={"c": {"max": 4}, "d": {"min": 5}}, variables={"x": {"p": 1, "c": 1, "d": 1}})
    with pytest.raises(ValueError, match="bounded"):
        J.Solve(bounded, full=True).unbounded()
    with pytest.raises(ValueError, match="infeasible"):
        J.Solve(infeasible, full=True).unbounded()
    with pytest.raises(ValueError, match="integer or binary"):
        J.Solve(dict(EXAMPLE, ints={"x": 1}), full=True).unbounded()
    with pytest.raises(ValueError, match="unrestricted"):
        J.Solve(dict(EXAMPLE, unrestricted={"x": 1}), full=True).unbounded()
    sol = J.Solve(strip_timeouts(EXAMPLE), full=True)
    sol._tableau.simplex()
    with pytest.raises(ValueError, match="edited or solved again"):
        sol.unbounded()

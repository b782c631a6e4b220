"""GPU checks of the two-objective frontier (DESIGN.md section 2g): k_price_objective's R2 and E, every breakpoint record
of jslp_frontier (theta, raw objective, direction entry, pivot row and column, labels), the stop, every point and the
end state are bit-identical to oracle/frontier.py run from the same downloaded optimal tableau, after solves on
engines 0, 1, 2 and 4; the pricing at its row-block and column-tile edges; the call leaves the tableau as it was; and
Frontier() equals the oracle's Frontier()."""
import hashlib

import numpy as np
import pytest

from conftest import load_bundle
from helpers import strip_timeouts

pytestmark = pytest.mark.gpu
BUNDLE = load_bundle()
ENGINES = (0, 1, 2, 4)
BERLIN = {"optimize": {"capacity": "max", "cost": "min"},
          "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
          "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                        "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _soft(jm):
    return any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())


CONTINUOUS = [f for f in BUNDLE["fixtures"] if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"]))
              and isinstance(f["model"].get("optimize"), str)]


def _solve(it, engine, precision=1e-8):
    from jslpsolver_b200 import _lib
    from jslpsolver_b200.tableau import GpuTableau
    g = GpuTableau(precision)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, it.integerIndices, it.optionalCosts)
    g.set_option(_lib.OPT_ENGINE, engine)
    g.simplex()
    return g


def _state_hash(g):
    g._cache.clear()
    h = hashlib.sha256()
    for a in (g.matrix2d(), g.varIndexByRow, g.varIndexByCol, g.optional_reduced_costs()):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def assert_frontier_matches(g, unrestricted, c2, cap, what, pricing_only=False):
    """Device against the restatement from the same tableau; returns the restatement's output."""
    from oracle import frontier as OF
    g._cache.clear()
    M, vr, vc = g.matrix2d(), np.array(g.varIndexByRow), np.array(g.varIndexByCol)
    before = _state_hash(g)
    want = OF.path(M, vr, vc, unrestricted, g.precision, c2, cap)
    got = g.frontier_path(c2, cap)
    assert _state_hash(g) == before, f"{what}: the tableau changed"
    assert np.array_equal(_bits(got["r2"]), _bits(want["r2"])), f"{what}: R2"
    assert np.array_equal(_bits(got["dir"]), _bits(want["dir"])), f"{what}: E"
    if pricing_only:
        return want
    n = len(want["records"])
    assert got["stop"] == want["stop"] and len(got["theta"]) == n, (what, got["stop"], want["stop"], len(got["theta"]), n)
    w = np.array([r[:3] for r in want["records"]], dtype=np.float64).reshape(n, 3)
    a = np.stack([got["theta"], got["obj_raw"], got["dobj"]], axis=1)
    bad = np.nonzero((_bits(a) != _bits(w)).any(axis=1))[0]
    assert len(bad) == 0, f"{what}: record {bad[:3].tolist()}: device {a[bad[:3]]} restatement {w[bad[:3]]}"
    assert np.array_equal(np.array([r[3:] for r in want["records"]], dtype=np.int64).reshape(n, 4),
                          got["rc_lbl"].astype(np.int64)), what
    assert got["n_points"] == len(want["points"]) == len(got["pt_break"]), (what, got["n_points"], len(want["points"]))
    for k, (rhs, vrow, at) in enumerate(want["points"]):
        assert int(got["pt_break"][k]) == at, (what, k)
        assert np.array_equal(_bits(got["pt_rhs"][k]), _bits(rhs)) and np.array_equal(got["pt_vrow"][k], vrow), (what, k)
    assert np.array_equal(_bits(got["end_rhs"]), _bits(want["end_rhs"])), what
    assert np.array_equal(got["end_vrow"], want["end_vrow"]), what
    return want


def _c2(m, rng, sense, fixed=()):
    sigma = 1.0 if sense == "max" else -1.0
    c2 = np.zeros(len(m.variables) + len(m.constraints))
    for v in m.variables:
        if v not in fixed:
            c2[v.index] = sigma * float(rng.integers(0, 21))
    return c2


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("fx", CONTINUOUS, ids=lambda f: f["file"])
def test_fixture_frontiers_bit_identical(fx, engine):
    """Each continuous fixture's optimum with a seeded second objective of both senses."""
    from jslpsolver_b200.model import Model, presolve
    m = Model().loadJson(strip_timeouts(fx["model"]))
    pr = presolve(m)
    if pr.isInfeasible:
        pytest.skip("decided by presolve")
    for v in pr.fixedVariables:
        v.cost = 0
    it = m.initial_tableau()
    g = _solve(it, engine)
    if not (g.feasible and g.bounded):
        pytest.skip("no optimum")
    rng = np.random.default_rng(len(m.variables))
    for sense in ("max", "min"):
        assert_frontier_matches(g, it.unrestricted, _c2(m, rng, sense, pr.fixedVariables), 4 * (g.height + g.width),
                                f"{fx['file']} {sense}")
    g.close()


def _multi_tableau(n, m, seed):
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    jm = problems.dense_packing_multi_model(n, m, 2, seed)
    model = Model().loadJson(dict(jm, optimize="profit", opType="max"))
    c2 = np.zeros(len(model.variables) + len(model.constraints))
    for v in model.variables:
        c2[v.index] = jm["variables"][v.id]["attr1"]
    return model.initial_tableau(), c2


@pytest.mark.parametrize("engine", ENGINES)
def test_tableau_beyond_shared_memory(engine):
    """dense_packing_multi_model at 121 x 151 and 333 x 257 (beyond shared memory): the whole path, max and min."""
    for n, m, seed in ((121, 151, 3), (333, 257, 5)):
        it, c2 = _multi_tableau(n, m, seed)
        g = _solve(it, engine)
        assert g.feasible and g.bounded
        want = assert_frontier_matches(g, it.unrestricted, c2, 4 * (g.height + g.width), f"{n}x{m} max")
        assert len(want["records"]) > 1
        assert_frontier_matches(g, it.unrestricted, -c2, 4 * (g.height + g.width), f"{n}x{m} min")
        g.close()


def test_config3_optimum():
    """The 2001 x 2001 benchmark LP re-solved on the device: R2 and E, then the first 40 breakpoints (two polls)."""
    from jslpsolver_b200 import problems
    n = m = 2000
    it = problems.dense_packing_lp_tableau(n, m, 12345)
    rng = np.random.default_rng(12345)  # attr1 of dense_packing_multi_model(2000, 2000, 2), drawn as it draws it
    rng.integers(1, 21, size=(m, n)); rng.integers(100, 501, size=m); rng.integers(1, 51, size=n)
    c2 = np.zeros(n + m)
    c2[m:] = rng.integers(1, 51, size=(1, n))[0]  # variables take labels m .. m + n - 1
    g = _solve(it, 0)
    assert g.feasible and g.bounded
    want = assert_frontier_matches(g, it.unrestricted, c2, 40, "config 3")
    assert len(want["records"]) == 40 and want["stop"] == 4
    g.close()


def _random_tableau(H, W, seed, zero_rows=()):
    """An uploaded (not optimal) tableau and a C2 with +-0 coefficients and whole row blocks skipped."""
    from jslpsolver_b200.tableau import GpuTableau
    rng = np.random.default_rng(seed)
    M = rng.standard_normal((H, W))
    M[rng.random((H, W)) < 0.1] = 0.0
    M[rng.random((H, W)) < 0.05] = -0.0
    labels = rng.permutation(H + W - 2).astype(np.int32)
    vcol = np.concatenate([[-1], labels[:W - 1]]).astype(np.int32)
    vrow = np.concatenate([[-1], labels[W - 1:]]).astype(np.int32)
    c2 = rng.standard_normal(H + W - 2) * 10.0
    c2[rng.random(H + W - 2) < 0.2] = 0.0
    c2[rng.random(H + W - 2) < 0.1] = -0.0
    for r in zero_rows:
        c2[vrow[r]] = 0.0 if r % 2 else -0.0
    g = GpuTableau(1e-8)
    g.upload(M, vrow, vcol)
    return g, c2


@pytest.mark.parametrize("H1", [1, 63, 64, 65, 128, 129, 300])
@pytest.mark.parametrize("W", [2, 127, 128, 129, 257])
def test_price_objective_at_its_edges(H1, W):
    """k_price_objective at row-block edges (H - 1 = 63, 64, 65, 128, 129 rows) and column-tile edges (127, 128, 129,
    257 columns), with +-0 coefficients and the second row block skipped entirely."""
    skipped = range(65, min(129, H1 + 1))
    g, c2 = _random_tableau(H1 + 1, W, 1000 * H1 + W, zero_rows=skipped)
    assert_frontier_matches(g, None, c2, 1, f"H-1={H1} W={W}", pricing_only=True)
    g.close()


def test_degenerate_path_with_zero_length_pieces():
    """max x + y with three optima at theta = 0 (x + y <= 4, x <= 3, y <= 3), second objective max x: the path pivots
    at theta = 0 before it moves, and those points drop out of the vertices."""
    import jslpsolver_b200 as J
    from oracle import frontier as OF
    jm = {"optimize": {"s": "max", "x1": "max"},
          "constraints": {"sum": {"max": 4}, "cx": {"max": 3}, "cy": {"max": 3}, "z": {"max": 10}},
          "variables": {"y": {"s": 1, "sum": 1, "cy": 1, "z": 1}, "x": {"s": 1, "x1": 1, "sum": 1, "cx": 1, "z": 1}}}
    res, det = OF.Frontier(jm)
    thetas = [r[0] for r in det["path"]["records"]]
    assert thetas[0] == 0.0 and det["path"]["records"][0][3] >= 0, thetas
    assert J.Frontier(jm) == res
    assert res["vertices"][0]["values"] == {"y": 1.0, "x": 3.0} and res["vertices"][0]["weight"] == {"from": 0.0, "to": 1.0}


def test_tableau_unchanged_and_other_tools_still_work():
    """After Frontier's path on a solved tableau: the tableau, labels and optional rows are as they were,
    jslp_parametric still matches its restatement and sensitivity() reports the same."""
    import jslpsolver_b200 as J
    from jslpsolver_b200 import problems
    from oracle import parametric as OP
    sol = J.Solve(problems.mixed_lp_model(60, 40, seed=12), full=True)
    assert sol.feasible and sol.bounded
    g = sol._tableau
    before, rep = _state_hash(g), sol.sensitivity()
    m = g.model
    c2 = _c2(m, np.random.default_rng(5), "max")
    g.frontier_path(c2, 4 * (g.height + g.width))
    assert _state_hash(g) == before and g.nOpt == 0
    assert sol.sensitivity() == rep
    v = next(v for v in m.variables if v.cost)
    sigma = -1.0 if m.isMinimization else 1.0
    g._cache.clear()
    M, vr, vc = g.matrix2d(), np.array(g.varIndexByRow), np.array(g.varIndexByCol)
    unres = np.zeros(g.nVars, dtype=np.uint8)
    want = OP.path(M, vr, vc, unres, g.precision, 1, [v.index], [sigma], float(v.cost), 3.0 * v.cost, 1000)
    got = g.parametric_path(1, [v.index], [sigma], float(v.cost), 3.0 * v.cost, 1000)
    assert np.array_equal(_bits(got["theta"]), _bits([r[0] for r in want["records"]])) and got["stop"] == want["stop"]
    assert _state_hash(g) == before


def _seeded_models():
    from jslpsolver_b200 import problems
    out = [("berlin", BERLIN)]
    for seed in range(3):
        jm = problems.dense_packing_multi_model(12 + seed, 9 + seed, 2, seed)
        out.append((f"dense{seed}", jm))
        out.append((f"dense{seed} min", dict(jm, optimize={"profit": "max", "attr1": "min"})))
        mx = problems.mixed_lp_model(10 + seed, 7 + seed, seed=200 + seed)
        rng = np.random.default_rng(seed)
        for v in mx["variables"].values():
            v["second"] = float(rng.integers(-5, 20))
        out.append((f"mixed{seed}", dict(mx, optimize={"objective": mx["opType"], "second": "min"})))
    return out


@pytest.mark.parametrize("name,jm", _seeded_models(), ids=[n for n, _ in _seeded_models()])
def test_frontier_end_to_end_equals_the_oracle(name, jm):
    import jslpsolver_b200 as J
    from oracle import frontier as OF
    try:
        want, _ = OF.Frontier(jm)
    except ValueError:
        with pytest.raises(ValueError, match="other way round"):
            J.Frontier(jm)
        return
    got = J.Frontier(jm)
    assert got == want, name
    if name == "berlin":
        assert [v["values"] for v in got["vertices"]] == [{"brit": 24.0, "yank": 20.0}, {"brit": 44.0, "yank": 0.0},
                                                          {"brit": 0.0, "yank": 0.0}]

"""GPU checks of the parametric path: every breakpoint record of jslp_parametric (theta, raw objective, direction
entry, pivot row and column, labels), the stop and the end state are bit-identical to oracle/parametric.py run from
the same downloaded optimal tableau, after solves with the automatic engine (whose ping-pong step leaves the result in
either buffer) and with the two-kernel engine; paths cross graph polls and stop at the cap; the call leaves the
tableau as it was; and Solution.parametric() equals the restatement's result."""
import hashlib

import numpy as np
import pytest

from conftest import load_bundle
from helpers import strip_timeouts

pytestmark = pytest.mark.gpu
BUNDLE = load_bundle()
ENGINES = {"auto": 0, "two_kernel": 1}
LONGEST = [0]  # most records seen in one path (paths beyond 32 cross a graph poll)


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


def assert_path_matches(g, unrestricted, kind, labels, signs, theta0, target, cap, what):
    from oracle import parametric as OP
    g._cache.clear()
    M, vr, vc = g.matrix2d(), np.array(g.varIndexByRow), np.array(g.varIndexByCol)
    want = OP.path(M, vr, vc, unrestricted, g.precision, kind, labels, signs, theta0, target, cap)
    got = g.parametric_path(kind, labels, signs, theta0, target, cap)
    n = len(want["records"])
    assert got["stop"] == want["stop"] and len(got["theta"]) == n, (what, got["stop"], want["stop"], len(got["theta"]), n)
    w = np.array([r[:3] for r in want["records"]], dtype=np.float64).reshape(n, 3)
    a = np.stack([got["theta"], got["obj_raw"], got["dobj"]], axis=1)
    bad = np.nonzero((_bits(a) != _bits(w)).any(axis=1))[0]
    assert len(bad) == 0, f"{what}: record {bad[:3].tolist()}: device {a[bad[:3]]} restatement {w[bad[:3]]}"
    assert np.array_equal(np.array([r[3:] for r in want["records"]], dtype=np.int64).reshape(n, 4),
                          got["rc_lbl"].astype(np.int64)), what
    assert np.array_equal(_bits(got["end_rhs"]), _bits(want["end_rhs"])), what
    assert np.array_equal(got["end_vrow"], want["end_vrow"]), what
    LONGEST[0] = max(LONGEST[0], n)
    return n


def _g(theta0, target):
    return 1.0 if target >= theta0 else -1.0


CONTINUOUS = [f for f in BUNDLE["fixtures"] if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"]))
              and isinstance(f["model"].get("optimize"), str)]


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("fx", CONTINUOUS, ids=lambda f: f["file"])
def test_fixture_paths_bit_identical(fx, engine):
    """Every row and every variable of each continuous fixture, both directions, to targets far past the current
    value (the 600-row fixture: every 10th)."""
    from jslpsolver_b200.model import Model, presolve
    m = Model().loadJson(strip_timeouts(fx["model"]))
    pr = presolve(m)
    if pr.isInfeasible:
        pytest.skip("decided by presolve")
    for v in pr.fixedVariables:
        v.cost = 0
    it = m.initial_tableau()
    g = _solve(it, ENGINES[engine])
    if not (g.feasible and g.bounded):
        pytest.skip("no optimum")
    sigma = -1.0 if m.isMinimization else 1.0
    every = 10 if len(m.constraints) > 100 else 1
    for k, con in enumerate(m.constraints[::every]):
        s = 1.0 if con.isUpperBound else -1.0
        for target in (con.rhs + 3.0 * max(1.0, abs(con.rhs)), con.rhs - 3.0 * max(1.0, abs(con.rhs))):
            assert_path_matches(g, it.unrestricted, 0, [con.index], [_g(con.rhs, target) * s], float(con.rhs),
                                float(target), 4 * (g.height + g.width), f"{fx['file']} row {con.index} -> {target}")
    for v in m.variables[::every]:
        if v in pr.fixedVariables:
            continue
        for target in (v.cost + 3.0 * max(1.0, abs(v.cost)), v.cost - 3.0 * max(1.0, abs(v.cost))):
            assert_path_matches(g, it.unrestricted, 1, [v.index], [_g(v.cost, target) * sigma], float(v.cost),
                                float(target), 4 * (g.height + g.width), f"{fx['file']} cost {v.id} -> {target}")
    g.close()


def _with_unrestricted(jm, every):
    jm = dict(jm)
    jm["unrestricted"] = {v: 1 for k, v in enumerate(jm["variables"]) if k % every == 0}
    return jm


SEEDED = {"dense 333x257": ("dense", 333, 257, 5, 6), "mixed 260x200": ("mixed", 260, 200, 14, 6),
          "mixed 60x40 unrestricted": ("mixed_free", 60, 40, 56, 6),
          "tall dense 40x10000": ("dense", 40, 10000, 8, 3), "config 3 dense 2000x2000": ("dense", 2000, 2000, 12345, 1)}


def _seeded_tableau(kind, n, m, seed):
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    if kind == "dense":
        return problems.dense_packing_lp_tableau(n, m, seed)
    jm = problems.mixed_lp_model(n, m, seed)
    return Model().loadJson(_with_unrestricted(jm, 6) if kind == "mixed_free" else jm).initial_tableau()


def _picks(g, it, n_each):
    """Binding rows with the largest duals and basic structural variables, with their current values."""
    g._cache.clear()
    M, vr, vc = g.matrix2d(), np.array(g.varIndexByRow), np.array(g.varIndexByCol)
    H0 = it.matrix.shape[0]
    slack_row = {int(it.varIndexByRow[r]): r for r in range(1, H0)}
    var_col = {int(it.varIndexByCol[c]): c for c in range(1, it.matrix.shape[1])}
    binding = sorted(((abs(M[0, c]), int(vc[c])) for c in range(1, M.shape[1]) if int(vc[c]) in slack_row), reverse=True)
    basic = [int(vr[r]) for r in range(1, M.shape[0]) if int(vr[r]) in var_col]
    rows = [(lab, slack_row[lab]) for _, lab in binding[:n_each]]
    cols = [(lab, var_col[lab]) for lab in basic[:n_each]]
    return rows, cols


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("case", list(SEEDED))
def test_seeded_paths_bit_identical(case, engine):
    """Seeded LPs: right-hand sides of binding rows to 4x and to 0, costs of basic variables to 2x and to 0; the
    config-3 tableau runs one path of each kind capped at 64 breakpoints."""
    kind, n, m, seed, n_each = SEEDED[case]
    it = _seeded_tableau(kind, n, m, seed)
    g = _solve(it, ENGINES[engine])
    assert g.feasible and g.bounded
    if kind == "mixed_free":
        assert it.unrestricted.any()
    cap = 64 if n >= 2000 else 4 * (g.height + g.width)
    rows, cols = _picks(g, it, n_each)
    # theta is measured in tableau units here (row sign and objective sense +1): the records do not depend on it
    for lab, r0 in rows:
        rhs = float(it.matrix[r0, 0])
        for target in ((4.0 * rhs,) if n >= 2000 else (4.0 * rhs + 1.0, 0.0)):
            assert_path_matches(g, it.unrestricted, 0, [lab], [_g(rhs, target)], rhs, target, cap, f"{case} row {lab}")
    for lab, c0 in cols:
        cost = float(it.matrix[0, c0])
        for target in ((2.0 * cost,) if n >= 2000 else (2.0 * cost + 1.0, 0.0)):
            assert_path_matches(g, it.unrestricted, 1, [lab], [_g(cost, target)], cost, target, cap, f"{case} cost {lab}")
    g.close()


def test_long_paths_and_the_cap():
    """A path of more than 32 breakpoints (more than one graph per poll) and the `limit` stop at a cap of 3."""
    it = _seeded_tableau("dense", 333, 257, 5)
    g = _solve(it, 0)
    rows, _ = _picks(g, it, 8)
    longest = 0
    for lab, r0 in rows:
        rhs = float(it.matrix[r0, 0])
        longest = max(longest, assert_path_matches(g, it.unrestricted, 0, [lab], [-1.0], rhs, -1e9, 10000, f"row {lab} down"))
        longest = max(longest, assert_path_matches(g, it.unrestricted, 0, [lab], [1.0], rhs, 1e9, 10000, f"row {lab} up"))
    assert max(longest, LONGEST[0]) > 32, longest
    lab, r0 = rows[0]
    n = assert_path_matches(g, it.unrestricted, 0, [lab], [-1.0], float(it.matrix[r0, 0]), -1e9, 3, "cap 3")
    assert n == 3 and g.parametric_path(0, [lab], [-1.0], float(it.matrix[r0, 0]), -1e9, 3)["stop"] == 4
    g.close()


def _state_hash(g):
    g._cache.clear()
    h = hashlib.sha256()
    for a in (g.matrix2d(), g.varIndexByRow, g.varIndexByCol):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


@pytest.mark.parametrize("engine", list(ENGINES))
def test_tableau_unchanged_and_sensitivity_still_works(engine):
    import jslpsolver_b200 as J
    from jslpsolver_b200 import problems
    s = J.Solver()
    s.engine = ENGINES[engine]
    sol = s.Solve(problems.mixed_lp_model(60, 40, seed=12), full=True)
    assert sol.feasible and sol.bounded
    g = sol._tableau
    before, rep = _state_hash(g), sol.sensitivity()
    name = next(c["name"] for c in rep["constraints"] if c["dual"] != 0)
    var = next(k for k, v in rep["variables"].items() if v["value"] > 0)
    side = next(c["type"] for c in rep["constraints"] if c["name"] == name and c["dual"] != 0)
    sides = [c["type"] for c in rep["constraints"] if c["name"] == name]
    kw = {"side": side} if len(sides) == 2 else {}
    sol.parametric(constraint=name, to=0.0, **kw)
    sol.parametric(variable=var, to=3.0 * rep["variables"][var]["cost"] + 1.0)
    assert _state_hash(g) == before
    assert sol.sensitivity() == rep


REPORT_MODELS = [(f["file"], f["model"]) for f in CONTINUOUS + [r for r in BUNDLE["readme"] if not (
    r["model"].get("ints") or r["model"].get("binaries") or _soft(r["model"])) and isinstance(r["model"].get("optimize"), str)]]


@pytest.mark.parametrize("engine", list(ENGINES))
def test_solution_parametric_equals_the_restatement(engine):
    """Solve(model, full=True).parametric() on every continuous model against the restatement run from the oracle's
    own solve (whose final tableau the parity tests pin to the device's), shaped with labels mapped to names."""
    import jslpsolver_b200 as J
    from oracle import parametric as OP
    from oracle import ref_model
    from oracle import sensitivity as S
    s = J.Solver()
    s.engine = ENGINES[engine]
    checked = 0
    for name, jm in REPORT_MODELS:
        jm = strip_timeouts(jm)
        if len(jm["constraints"]) > 100:
            continue
        osol = ref_model.solve_full(jm, fast_cycles=True)
        gsol = s.Solve(jm, full=True)
        if osol.tableau is None or not (osol.feasible and osol.bounded):
            continue
        model = osol.model
        M, (vr, vc) = osol.tableau.matrix(), osol.tableau.maps()
        unres = np.zeros(M.shape[0] + M.shape[1] - 2, dtype=np.uint8)
        for i in model.unrestrictedVariables:
            unres[i] = 1
        sigma = -1.0 if model.isMinimization else 1.0
        names = S.json_row_names(jm)
        single = [k for k, n in enumerate(names) if names.count(n) == 1]
        for k in single:
            con = model.constraints[k]
            target = con.rhs + 2.0 * max(1.0, abs(con.rhs))
            got = gsol.parametric(constraint=names[k], to=target)
            p = OP.path(M, vr, vc, unres, model.precision, 0, [con.index], [1.0 if con.isUpperBound else -1.0],
                        float(con.rhs), target, 4 * sum(M.shape))
            want = OP.result(p, sigma, float(con.rhs), target, float(M[0, 0]))
            assert [(pc["from"], pc["to"], pc["result"], pc["slope"]) for pc in got["pieces"]] == \
                [(pc["from"], pc["to"], pc["result"], pc["slope"]) for pc in want["pieces"]], (name, names[k])
            assert (got["stop"], got["end"], got["result"]) == (want["stop"], want["end"], want["result"]), name
            checked += 1
    assert checked >= 15, checked


def test_berlin_known_answers_on_the_device():
    import jslpsolver_b200 as J
    berlin = {"optimize": "capacity", "opType": "max",
              "constraints": {"plane": {"max": 44}, "person": {"max": 512}, "cost": {"max": 300000}},
              "variables": {"brit": {"capacity": 20000, "plane": 1, "person": 8, "cost": 5000},
                            "yank": {"capacity": 30000, "plane": 1, "person": 16, "cost": 9000}}}
    sol = J.Solve(berlin, full=True)

    def nonzero(out):
        return [(pc["from"], pc["to"], pc["result"]["to"], pc["slope"]) for pc in out["pieces"] if pc["to"] != pc["from"]]

    assert nonzero(sol.parametric(constraint="person", to=0)) == [(512.0, 352.0, 880000.0, 1250.0), (352.0, 0.0, 0.0, 2500.0)]
    out = sol.parametric(constraint="person", to=1000)
    assert nonzero(out) == [(512.0, 1000.0, 1080000.0, 0.0)] and out["result"] == 1080000.0
    assert nonzero(sol.parametric(variable="brit", to=40000)) == [(20000.0, 30000.0, 1320000.0, 24.0),
                                                                   (30000.0, 40000.0, 1760000.0, 44.0)]
    assert nonzero(sol.parametric(variable="brit", to=10000)) == [(20000.0, 15000.0, 960000.0, 24.0),
                                                                   (15000.0, 10000.0, 960000.0, 0.0)]
    with pytest.raises(ValueError, match="no constraint named"):
        sol.parametric(constraint="nope", to=1)

"""GPU checks of the irreducible infeasible subset (DESIGN.md section 2c): jslp_feasibility_batch gives the oracle's
phase-1 verdict and pivot count set by set (shared-memory batch, HBM path, sets that overflow the in-kernel log cap,
cycling sets), Solution.iis() equals the oracle's literal filter at several speculation widths, it leaves the user's
tableau untouched, and the error cases raise."""
import hashlib

import numpy as np
import pytest

from conftest import load_bundle
from helpers import strip_timeouts

pytestmark = pytest.mark.gpu
BUNDLE = load_bundle()


def _soft(jm):
    return any(isinstance(s, dict) and ("weight" in s or "priority" in s) for s in jm["constraints"].values())


CONTINUOUS = [f for f in BUNDLE["fixtures"] if not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"]))
              and isinstance(f["model"].get("optimize"), str)]
INFEASIBLE = [f for f in BUNDLE["fixtures"] if f.get("expects", {}).get("feasible") is False
              and not (f["model"].get("ints") or f["model"].get("binaries") or _soft(f["model"]))]


def _model(jm):
    from jslpsolver_b200.model import Model
    return Model().loadJson(strip_timeouts(jm))


def _gpu(it, precision, engine=None, options=None):
    from jslpsolver_b200 import _lib
    from jslpsolver_b200.tableau import GpuTableau
    g = GpuTableau(precision)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted)
    if engine is not None:
        g.set_option(_lib.OPT_ENGINE, engine)
    for k, v in (options or {}).items():
        g.set_option(k, v)
    g.save()
    return g


def _random_sets(H, n, rng, p=0.7):
    sets = [list(range(1, H)), []]
    for _ in range(n):
        sets.append([r for r in range(1, H) if rng.random() < p])
    return sets


def _check_batch(it, precision, sets, what, engine=None, options=None):
    from oracle import iis as O
    g = _gpu(it, precision, engine, options)
    H = it.matrix.shape[0]
    keep = np.zeros((len(sets), H), dtype=np.uint8)
    for i, s in enumerate(sets):
        keep[i, s] = 1
    before = g.matrix2d().copy()
    verdict, pivots = g.feasibility_batch(keep)
    want = [O.test(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, precision, s) for s in sets]
    for i, (v, p) in enumerate(want):
        assert (int(verdict[i]), int(pivots[i])) == (v, p), f"{what}: set {i} ({len(sets[i])} rows): device " \
            f"{(int(verdict[i]), int(pivots[i]))} oracle {(v, p)}"
    assert np.array_equal(g.matrix2d().view(np.uint64), before.view(np.uint64)), f"{what}: tableau != snapshot"
    g.close()
    return [v for v, _ in want]


@pytest.mark.parametrize("path", ["k2", "hbm"])
@pytest.mark.parametrize("fx", CONTINUOUS, ids=lambda f: f["file"])
def test_fixture_subsets_match_oracle(fx, path):
    m = _model(fx["model"])
    it = m.initial_tableau()
    sets = _random_sets(it.matrix.shape[0], 12, np.random.default_rng(7))
    _check_batch(it, m.precision, sets, fx["file"], engine=None if path == "k2" else 2)


SEEDED = {"dense 30x20": ("dense", 30, 20, 1), "mixed 40x30": ("mixed", 40, 30, 11), "mixed 90x60": ("mixed", 90, 60, 13),
          "mixed 40x30 unrestricted": ("mixed_free", 40, 30, 12), "random 40x30": ("random", 40, 30, 5),
          "random 30x25 unrestricted": ("random_free", 30, 25, 6),
          # root heights 32, 33, 64, 65 (cost row included): the keep mask fills one / spills into a second 32-bit word
          "mixed 20x31": ("mixed", 20, 31, 31), "mixed 20x32": ("mixed", 20, 32, 32),
          "mixed 24x63": ("mixed", 24, 63, 33), "mixed 24x64": ("mixed", 24, 64, 34)}


def _seeded(kind, n, mcons, seed):
    from jslpsolver_b200 import problems
    if kind == "dense":
        jm = problems.dense_packing_lp_model(n, mcons, seed)
        jm["constraints"] = {k: ({"min": v["max"] * 0.05} if i % 3 == 0 else v)
                             for i, (k, v) in enumerate(jm["constraints"].items())}
    elif kind.startswith("mixed"):
        jm = problems.mixed_lp_model(n, mcons, seed, frac_min=0.5)
    else:
        jm = problems.random_lp_model(n, mcons, seed)
    if kind.endswith("free"):
        jm["unrestricted"] = {v: 1 for k, v in enumerate(jm["variables"]) if k % 4 == 0}
    return jm


@pytest.mark.parametrize("path", ["k2", "hbm"])
@pytest.mark.parametrize("name", list(SEEDED))
def test_seeded_subsets_match_oracle(name, path):
    m = _model(_seeded(*SEEDED[name]))
    it = m.initial_tableau()
    sets = _random_sets(it.matrix.shape[0], 40 if path == "k2" else 8, np.random.default_rng(3), p=0.8)
    _check_batch(it, m.precision, sets, name, engine=None if path == "k2" else 2)


@pytest.mark.parametrize("size", ["k2 150x120", "hbm 550x600"])
def test_planted_subsets_match_oracle(size):
    from jslpsolver_b200 import problems
    n, mcons = (150, 120) if size.startswith("k2") else (550, 600)
    m = _model(problems.planted_infeasible_model(n, mcons, 6, 21))
    it = m.initial_tableau()
    sets = _random_sets(it.matrix.shape[0], 24 if size.startswith("k2") else 3, np.random.default_rng(4), p=0.9)
    _check_batch(it, m.precision, sets, size)


def test_log_cap_overflow_reruns_on_hbm():
    """A node log cap of 4 entries sends every set with more phase-1 pivots to the HBM path; results are unchanged."""
    from jslpsolver_b200 import _lib
    m = _model(_seeded(*SEEDED["mixed 90x60"]))
    it = m.initial_tableau()
    sets = _random_sets(it.matrix.shape[0], 16, np.random.default_rng(9), p=0.85)
    _check_batch(it, m.precision, sets, "log cap 4", options={_lib.OPT_NODE_LOG_CAP: 4})


@pytest.mark.parametrize("path", ["k2", "hbm"])
def test_cycling_sets_are_undecided(path):
    """ChenhuaWANG22_2's phase 1 cycles on the whole LP and on most one-row-smaller subsets: the oracle's cycle check
    stops them, and the device must call them undecided with the same pivot count."""
    fx = [f for f in CONTINUOUS if f["file"] == "ChenhuaWANG22_2.json"][0]
    m = _model(fx["model"])
    it = m.initial_tableau()
    H = it.matrix.shape[0]
    sets = [list(range(1, H))] + [[r for r in range(1, H) if r != s] for s in range(1, H)]
    sets += _random_sets(H, 20, np.random.default_rng(2), p=0.9)
    verdicts = _check_batch(it, m.precision, sets, "ChenhuaWANG22_2", engine=None if path == "k2" else 2)
    assert verdicts.count(2) >= 10


def _solution(jm):
    from jslpsolver_b200 import Solve
    return Solve(jm, full=True)


def _oracle_iis(sol):
    from oracle import iis as O
    m = sol._tableau.model
    it = m.initial_tableau()
    kept, irreducible, _ = O.iis(it, m.precision)
    cons = []
    for r in kept:
        c = m.constraints[r - 1]
        cons.append({"name": c.name if c.name is not None else c.index, "type": "max" if c.isUpperBound else "min",
                     "rhs": c.rhs})
    return cons, irreducible


def _iis_cases():
    from jslpsolver_b200 import problems
    cases = [(f["file"], strip_timeouts(f["model"])) for f in INFEASIBLE if f["file"] != "ChenhuaWANG22_2.json"]
    seed, n = 0, 0
    while n < 8 and seed < 400:
        rng = np.random.default_rng(seed)
        jm = problems.random_lp_model(int(rng.integers(6, 41)), int(rng.integers(5, 31)), seed=1000 + seed)
        from oracle import iis as O
        mm = _model(jm)
        it = mm.initial_tableau()
        if O.start_set(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, mm.precision)[2] == O.INFEASIBLE:
            cases.append((f"random seed {seed}", jm))
            n += 1
        seed += 1
    cases.append(("planted k2 150x120", problems.planted_infeasible_model(150, 120, 6, 31)))
    cases.append(("planted hbm 550x600", problems.planted_infeasible_model(550, 600, 5, 32)))
    return cases


@pytest.mark.parametrize("width", [1, 8, None], ids=["w1", "w8", "default"])
def test_iis_matches_oracle_literal_filter(width):
    from jslpsolver_b200.iis import compute
    for label, jm in _iis_cases():
        sol = _solution(jm)
        assert not sol.feasible, label
        want, irreducible = _oracle_iis(sol)
        got = sol.iis() if width is None else compute(sol, width=width, prepass=width > 1)
        assert got["constraints"] == want and got["irreducible"] == irreducible, label
        names = []
        for c in want:
            if c["name"] not in names:
                names.append(c["name"])
        assert got["names"] == names and got["lps"] >= 1 + len(want), label
        if label.startswith("planted"):
            assert sorted(c["name"] for c in got["constraints"]) == sorted(f"conflict{p}" for p in range(len(want)))
        if label == "Infeasible Berlin Air Lift Problem.json":
            assert got["constraints"] == [{"name": "brit", "type": "min", "rhs": 13}]


def test_iis_leaves_the_user_tableau_untouched():
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    jm = problems.planted_infeasible_model(40, 30, 4, 3)
    jm["options"] = {"presolve": False}  # presolve would decide it before any tableau is uploaded
    m = Model().loadJson(jm)
    sol = m.solve()
    assert not sol.feasible and m.tableau.handle is not None
    t = m.tableau
    digest = hashlib.sha256(t.matrix2d().tobytes()).hexdigest()
    vrow, vcol, version = t.varIndexByRow.copy(), t.varIndexByCol.copy(), t._version
    out = sol.iis()
    assert sorted(out["names"]) == [f"conflict{p}" for p in range(4)]
    t._cache.clear()
    assert hashlib.sha256(t.matrix2d().tobytes()).hexdigest() == digest and t._version == version
    assert np.array_equal(t.varIndexByRow, vrow) and np.array_equal(t.varIndexByCol, vcol)
    assert sol.iis() == out  # and it can be asked again


def test_iis_value_errors():
    from jslpsolver_b200 import Solve
    from jslpsolver_b200.model import Model
    lp = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Berlin Air Lift Problem.json"][0]["model"])
    with pytest.raises(ValueError, match="feasible"):
        Solve(lp, full=True).iis()
    cyc = strip_timeouts([f for f in CONTINUOUS if f["file"] == "ChenhuaWANG22_2.json"][0]["model"])
    sol = Solve(cyc, full=True)
    assert not sol.feasible
    with pytest.raises(ValueError, match="cycles"):
        sol.iis()
    bad = strip_timeouts([f for f in INFEASIBLE if f["file"] == "Infeasible 1.json"][0]["model"])
    m = Model().loadJson(bad)
    sol = m.solve()
    assert not sol.feasible and m.tableau.handle is not None
    m.tableau.simplex()  # solved again after this solution
    with pytest.raises(ValueError, match="edited or solved again"):
        sol.iis()
    with pytest.raises(ValueError, match="integer or binary"):
        Solve(dict(bad, ints={"x": 1}), full=True).iis()

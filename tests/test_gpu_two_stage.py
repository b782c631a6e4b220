"""GPU checks of two-stage stochastic LPs (DESIGN.md section 2u): jslp_recourse_batch equals jslp_scenario_batch on the
same edits bit for bit, and its cert_rhs and alpha equal the restatement's bit for bit, on the shared-memory batch, on a
recourse tableau too tall for shared memory, on engine 2 and with the node log cap at 4 (every case redone on the
single-tableau path); alpha at k_recourse_alpha's tile edges; TwoStage() equals the restatement key for key on engines 0
and 2; and the caller's tableau is left as it was."""
import math

import numpy as np
import pytest

import two_stage_models as TM
import two_stage_oracle as TO

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _setup(model, cases, first, p, engine=0, options=None, x=None):
    """(device tableau of the recourse model at the plan x, oracle backend over the same tableau, Cases, x)."""
    from jslpsolver_b200 import _lib, two_stage as TS
    from jslpsolver_b200.solver import Solver
    pb = TS.Problem(TS._one_objective(model), first, TS._probabilities(p, len(cases)), None)
    x = [1.0 + j for j in range(len(pb.first))] if x is None else x
    s = Solver()
    s.engine = engine
    s.options = dict(options or {})
    dev = TS._Device(s, None)
    m, _ = dev.recourse(pb.recourse_json(x))
    orc = TO.Oracle()
    orc.recourse(pb.recourse_json(x))
    cs = TS.Cases(pb, m, cases)
    return dev, orc, cs, x


def _compare(dev, orc, cs, x):
    edits, offsets = cs.edits(x)
    before = dev.tab.matrix2d().copy(), dev.tab.varIndexByRow.copy(), dev.tab.varIndexByCol.copy()
    got = dev.batch(edits, offsets, cs.rows, cs.signed)
    dev.tab._edited()
    after = dev.tab.matrix2d(), dev.tab.varIndexByRow, dev.tab.varIndexByCol
    assert np.array_equal(_bits(before[0]), _bits(after[0])) and all(np.array_equal(a, b) for a, b in
                                                                        zip(before[1:], after[1:]))
    plain = dev.tab.scenario_batch(edits, offsets, check_cycles=True)
    for k in ("status", "p1", "p2", "vrow"):
        assert np.array_equal(got[k], plain[k]), k
    for k in ("eval_raw", "rhs"):
        assert np.array_equal(_bits(got[k]), _bits(plain[k])), k
    want = orc.batch(edits, offsets, cs.rows, cs.signed)
    for k in ("status", "p1", "p2", "vrow"):
        assert np.array_equal(got[k], want[k]), k
    for k in ("eval_raw", "rhs", "cert_rhs", "alpha"):
        assert np.array_equal(_bits(got[k]), _bits(want[k])), k
    return got


CASES = [(seed, kw) for seed in range(3) for kw in ({}, {"per_case_t": True}, {"complete": False})]


@pytest.mark.parametrize("seed,kw", CASES)
@pytest.mark.parametrize("engine,options", [(0, None), (2, None), (0, {14: 4})])
def test_recourse_batch_matches_scenarios_and_restatement(seed, kw, engine, options):
    model, cases, first, p = TM.capacity(seed, n_cases=24, **kw)
    dev, orc, cs, x = _setup(model, cases, first, p, engine, options)
    try:
        got = _compare(dev, orc, cs, x)
        if kw.get("complete") is False:
            got = _compare(dev, orc, cs, [0.0] * len(x))  # demand beyond zero capacity: Farkas rows
            assert (got["status"] == 1).any() and np.isfinite(got["cert_rhs"][got["status"] == 1]).all()
    finally:
        dev.close()


def test_tall_recourse_tableau():
    """Second-stage rows beyond shared memory: every case runs on the single-tableau path."""
    model, cases, first, p = TM.capacity(7, n_first=4, n_second=260, n_cases=6, per_case_t=True)
    dev, orc, cs, x = _setup(model, cases, first, p)
    try:
        assert dev.tab.height * dev.tab.width * 8 > 232448
        _compare(dev, orc, cs, x)
    finally:
        dev.close()


@pytest.mark.parametrize("n_first,n_cases", [(31, 7), (32, 8), (33, 9), (1, 1), (64, 17)])
def test_alpha_tile_edges(n_first, n_cases):
    model, cases, first, p = TM.capacity(3, n_cases=n_cases)
    dev, orc, cs, x = _setup(model, cases, first, p)
    try:
        rng = np.random.default_rng(n_first)
        for tech in (rng.standard_normal((len(cs.rows), n_first)),
                     rng.standard_normal((n_cases, len(cs.rows), n_first))):
            edits, offsets = cs.edits(x)
            got = dev.batch(edits, offsets, cs.rows, tech)
            want = orc.batch(edits, offsets, cs.rows, tech)
            assert got["alpha"].shape == (n_cases, n_first)
            assert np.array_equal(_bits(got["alpha"]), _bits(want["alpha"]))
    finally:
        dev.close()


def test_refusals():
    from jslpsolver_b200 import JslpError
    model, cases, first, p = TM.capacity(0)
    dev, orc, cs, x = _setup(model, cases, first, p)
    try:
        edits, offsets = cs.edits(x)
        for rows in ([-1] + cs.rows[1:], [cs.rows[0]] * 2 + cs.rows[2:], [10 ** 6] + cs.rows[1:]):
            with pytest.raises(JslpError):
                dev.batch(edits, offsets, rows, cs.signed)
        assert dev.batch(edits, offsets, [], np.zeros((0, 3)))["alpha"].tolist() == [[0.0] * 3] * len(cases)
    finally:
        dev.close()


FIXTURES = [("farmer", TM.FARMER, TM.FARMER_CASES, TM.FARMER_FIRST, None)] + [
    (f"capacity{seed}{sorted(kw)}", *TM.capacity(seed, **kw)) for seed, kw in
    [(s, kw) for s in range(4) for kw in ({}, {"per_case_t": True}, {"complete": False},
                                          {"max_sense": True, "per_case_t": True})] + [(4, {"complete": False})]]


@pytest.mark.parametrize("engine", [0, 2])
@pytest.mark.parametrize("name,model,cases,first,p", FIXTURES, ids=[f[0] for f in FIXTURES])
def test_two_stage_equals_restatement(engine, name, model, cases, first, p):
    from jslpsolver_b200.solver import Solver
    s = Solver()
    s.engine = engine
    got = s.TwoStage(model, cases, first, p)
    want = TO.TwoStage(model, cases, first, p)
    assert got["launches"] > 0
    got.pop("launches"), want.pop("launches")
    assert got.keys() == want.keys()
    for k in got:
        if isinstance(got[k], float) and math.isnan(got[k]):
            assert math.isnan(want[k])
        else:
            assert got[k] == want[k], k

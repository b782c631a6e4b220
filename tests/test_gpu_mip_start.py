"""MIP starts (DESIGN.md section 2t) on the device against tests/mip_start_oracle.py, bit for bit: node log, evaluation,
best cuts, final column 0 and row labels, and every start's status, evaluation, node count and pivots, at speculation
widths 1, 16 and the default, on engines 0 and 2, with node slots off and auto; on a knapsack whose start nodes are
beyond shared memory; with keep_solutions, tolerance > 0, useMIRCuts, a node pivot-log cap
of 2 and max_nodes reached with the seed still the incumbent.  jslp_branch_and_cut_start with no starts equals
jslp_branch_and_cut."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import pytest

import mip_start_oracle as MSO
import pool_oracle as PO
from helpers import strip_timeouts
from conftest import load_bundle
from jslpsolver_b200 import _lib, problems

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _oracle_lib():
    from oracle import ref_model
    ref_model.build_oracle()


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.int64)


def _plain(jm: dict) -> bool:
    tol = jm.get("tolerance") or (jm.get("options") or {}).get("tolerance")
    return (bool(jm.get("ints") or jm.get("binaries")) and isinstance(jm.get("optimize"), str) and not tol
            and len(jm["variables"]) <= 40 and not any(
                isinstance(c, dict) and (c.get("weight") is not None or c.get("priority") is not None)
                for c in jm["constraints"].values()))


FIXTURES = [strip_timeouts(fx["model"]) for fx in load_bundle()["fixtures"] if _plain(fx["model"])]
FAMILIES = [problems.knapsack_mip_model(12, 4, seed=1), problems.knapsack_mip_model(16, 6, seed=2),
            problems.random_mip_model(14, 8, seed=3), problems.random_mip_model(18, 10, seed=5),
            problems.set_cover_model(12, 10, seed=4), problems.half_tie_mip_model(12, seed=6)]
# 133 x 129: the root and the early tree nodes fit shared memory, the empty knapsack's node (128 cut rows) does not
BIG = problems.knapsack_mip_model(128, 4, seed=7)


def starts_of(jm: dict) -> list:
    """The cold optimum's plan, the second plan of the pool, a partial plan and an infeasible plan, in one call."""
    cold, _, _ = MSO.solve(jm)
    ints = [k for k in jm["variables"] if (jm.get("ints") or {}).get(k) or (jm.get("binaries") or {}).get(k)]
    plan = {k: v for k, v in cold.items() if k in jm["variables"]}
    out = [plan, {**plan, **{v: None for v in ints[::2]}}, {v: -1 for v in ints}, dict(cold)]
    if len(ints) <= 20:
        sols = PO.pool(jm, k=2)["solutions"]
        if len(sols) == 2:
            out.insert(1, sols[1]["values"])
    return out


def run(jm: dict, start, *, width=0, engine=0, slots=None, options=None, max_nodes=0, start_nodes=1000):
    import jslpsolver_b200 as J
    S = J.Solver()
    S.max_spec_batch, S.engine, S.node_slots, S.options = width, engine, slots, dict(options or {})
    m = S._instance(jm, None)
    m.max_nodes = max_nodes
    sol = m.solve(start=start, start_nodes=start_nodes)
    S._finish(m, sol, True)
    return m, sol, S._simplified(sol)


def same(m, sol, simplified, ref):
    simp, report, res = ref
    t = m.tableau
    gl, ol = t.node_log(), res["node_log"]
    assert gl.shape == ol.shape, (gl.shape, ol.shape)
    for i in range(len(ol)):
        a, b = gl[i], ol[i]
        assert all(a[k] == b[k] for k in (0, 1, 2, 4, 5, 7)) and bits(a[6]) == bits(b[6]), (i, a, b)
        assert bits(a[3]) == bits(b[3]), (i, a, b)
    st, fin = t.lastBnbStatus, res["o"].state()
    assert bits(st.evaluation) == bits(fin.evaluation)
    assert (st.feasible, st.bounded, st.iterations, bool(st.is_integral)) == \
        (fin.feasible, fin.bounded, res["iterations"], res["is_integral"])
    assert t.bestCuts == res["best_cuts"]
    assert np.array_equal(bits(t.rhs_column()), bits(res["o"].matrix()[:, 0]))
    assert np.array_equal(t.varIndexByRow, res["o"].maps()[0])
    assert len(t.lastStartStatus) == len(res["starts"])
    for g, o in zip(t.lastStartStatus, res["starts"]):
        assert (g.status, g.nodes, g.pivots, g.n_cuts) == (o["status"], o["nodes"], o["pivots"], o["n_cuts"])
        assert (math.isnan(g.evaluation) and math.isnan(o["evaluation"])) or bits(g.evaluation) == bits(o["evaluation"])
    assert sol.mipStart == report
    assert simplified == simp
    sols = res["solutions"]
    assert st.n_solutions == len(sols)
    L = t.context.lib
    for i, (ev, rhs, vrow) in enumerate(sols):
        e, h = C.c_double(), C.c_int32()
        _lib.check(L.jslp_bnb_solution(t._h(), i, C.byref(e), C.byref(h), None, None, 0))
        gv, gr = np.empty(h.value, dtype=np.int32), np.empty(h.value, dtype=np.float64)
        _lib.check(L.jslp_bnb_solution(t._h(), i, None, None, gv.ctypes.data, gr.ctypes.data, h.value))
        assert bits(e.value) == bits(ev) and np.array_equal(gv, vrow) and np.array_equal(bits(gr), bits(rhs))


CONFIGS = [(1, 0, None), (16, 0, None), (0, 0, None), (0, 2, None), (0, 2, 0), (16, 2, 0), (1, 2, None)]
MODELS = FAMILIES + FIXTURES


@pytest.mark.parametrize("k", range(len(MODELS)))
def test_device_equals_the_restatement(k):
    jm = MODELS[k]
    start = starts_of(jm)
    ref = MSO.solve(jm, start)
    for width, engine, slots in CONFIGS:
        same(*run(jm, start, width=width, engine=engine, slots=slots), ref)


@pytest.mark.parametrize("variant", ["keep_solutions", "tolerance", "mir", "log_cap", "max_nodes", "start_nodes"])
def test_device_equals_the_restatement_under_options(variant):
    base = problems.knapsack_mip_model(16, 6, seed=2)
    jm, kw, rkw = dict(base), {}, {}
    if variant == "keep_solutions":
        jm["options"] = {"keep_solutions": True}
    elif variant == "tolerance":
        jm["tolerance"] = 0.05
    elif variant == "mir":
        jm["options"] = {"useMIRCuts": True}
    elif variant == "log_cap":
        kw["options"] = {_lib.OPT_NODE_LOG_CAP: 2}
    elif variant == "max_nodes":
        kw["max_nodes"] = rkw["max_nodes"] = 3
    else:
        kw["start_nodes"] = rkw["start_nodes"] = 2
    start = starts_of(base)
    ref = MSO.solve(jm, start, **rkw)
    if variant == "max_nodes":
        assert ref[1]["seed"] is not None and not ref[1]["improved"]  # the seed is still the incumbent
    for width, engine, slots in [(1, 0, None), (0, 0, None), (0, 2, None)]:
        same(*run(jm, start, width=width, engine=engine, slots=slots, **kw), ref)


@pytest.mark.parametrize("width, engine, slots", [(1, 0, None), (16, 0, None), (0, 0, None), (0, 0, 0), (0, 2, None)])
def test_start_nodes_beyond_shared_memory(width, engine, slots):
    start = [{}, {k: None for k in BIG["variables"]}]  # the empty knapsack, and the root's own dive
    ref = _big_ref()
    assert ref[1]["starts"][0]["status"] in ("seed", "feasible")
    same(*run(BIG, start, width=width, engine=engine, slots=slots, max_nodes=20, start_nodes=50), ref)


_BIG = []


def _big_ref():
    if not _BIG:
        _BIG.append(MSO.solve(BIG, [{}, {k: None for k in BIG["variables"]}], max_nodes=20, start_nodes=50))
    return _BIG[0]


@pytest.mark.parametrize("k", [0, 2, 4, 5])
def test_no_starts_equals_branch_and_cut(k):
    import jslpsolver_b200 as J
    jm = FAMILIES[k]
    out = []
    for start in (None, []):
        m = J.Solver()._instance(jm, None)
        m.presolveResult = None
        m.solve() if start is None else m.solve(start=start)
        t = m.tableau
        st = t.lastBnbStatus
        out.append((t.node_log().tobytes(), st.feasible, st.iterations, st.nodes_evaluated, st.pivots,
                    bits(st.evaluation), st.kernel_launches, t.bestCuts, t.rhs_column().tobytes()))
    assert out[0] == out[1]

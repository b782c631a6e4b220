"""The caller's side of the six analysis batches that run sets of LPs on the node kernel (jslp_feasibility_batch,
jslp_conflict_batch, jslp_column_batch, jslp_scenario_batch, jslp_pool_batch, jslp_target_batch; DESIGN.md section
2e).  After one call that mixes resident, too-tall and redone sets wherever the entry point allows it, on engines 0 and
2 and with a node log cap of 2, the caller's tab is what a twin tab that never ran the call shows: matrix bits, labels,
dimensions and pivot log; the jslp_save snapshot that restore() brings back; and the scalar Tableau state a later
simplex() reports.  The batches over the snapshot leave the tableau equal to it, so their twin runs restore() instead.
Every argument refusal reports its message word for word."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import conflict_oracle as O
from jslpsolver_b200 import _lib, problems

pytestmark = pytest.mark.gpu

CONFIGS = [(0, None), (0, 2), (2, None)]  # (engine, node log cap)
CONFIG_IDS = ["engine0", "engine0-logcap2", "engine2"]
MIP = problems.planted_integer_conflict_model(30, 40, 4, 3)
TALL_CUTS = 1000  # cut rows that take a 41 x 31 tableau beyond one CTA's shared memory


def _tab(jm: dict, engine: int = 0, log_cap=None, save: bool = True):
    """jm's initial tableau, saved (the snapshot the batches read), then solved: the caller's own tableau, pivot log
    and scalar state."""
    from jslpsolver_b200.model import Model
    from jslpsolver_b200.tableau import GpuTableau
    m = Model().loadJson(jm)
    g = GpuTableau(m.precision)
    g.engine = engine
    g.options[_lib.OPT_PIVOT_LOG_CAP] = 1 << 20
    if log_cap:
        g.options[_lib.OPT_NODE_LOG_CAP] = log_cap
    g.setModel(m)
    if save:
        g.save()
    g.simplex()
    return g


def _seen(g) -> dict:
    g._refresh_dims()
    M = np.ascontiguousarray(g.matrix2d())
    return {"dims": (g.width, g.height, g.nVars, g.lastElementIndex), "matrix": M.view(np.uint64).tobytes(),
            "vrow": g.varIndexByRow.tobytes(), "vcol": g.varIndexByCol.tobytes(), "log": g.pivot_log().tobytes()}


def _status(st) -> tuple:
    out = []
    for name, ty in st._fields_:
        if name in ("gpu_ms", "kernel_launches"):
            continue
        v = getattr(st, name)
        out.append(int(np.float64(v).view(np.uint64)) if ty is C.c_double else v)
    return tuple(out)


def _after(g) -> dict:
    """What the caller sees of its tab now, after a pivot and restore() (the snapshot), and after a simplex() from
    there (the scalar state it starts from and the pivot log it appends to)."""
    out = {f"now {k}": v for k, v in _seen(g).items()}
    M = g.matrix2d()
    r, c = np.argwhere(np.abs(M[1:, 1:]) > 1e-3)[0]
    g.pivot(int(r) + 1, int(c) + 1)
    g.restore()
    out.update({f"restored {k}": v for k, v in _seen(g).items()})
    g.simplex()
    out.update({f"re-solved {k}": v for k, v in _seen(g).items()})
    out["re-solved status"] = _status(g.lastStatus)
    return out


def assert_untouched(jm: dict, engine: int, log_cap, call, over_snapshot: bool = True):
    a, b = _tab(jm, engine, log_cap), _tab(jm, engine, log_cap)
    try:
        call(a)
        if over_snapshot:
            b.restore()
        got, want = _after(a), _after(b)
        for k in want:
            assert got[k] == want[k], f"engine {engine}, log cap {log_cap}: {k} differs from the twin's"
    finally:
        a.close()
        b.close()


# ---- the caller's tab -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine, log_cap", CONFIGS, ids=CONFIG_IDS)
def test_feasibility_batch_leaves_the_caller_tab(engine, log_cap):
    # 401 x 151: one CTA holds about 180 rows, so the whole tableau and set 5 are too tall and the others fit
    jm = problems.planted_infeasible_model(150, 400, 4, 3)

    def call(g):
        assert (g.height, g.width) == (401, 151)
        rng = np.random.default_rng(1)
        keep = (rng.random((24, g.height)) < rng.uniform(0.05, 0.35, size=(24, 1))).astype(np.uint8)
        keep[0] = 1
        keep[5] = rng.random(g.height) < 0.6
        g.feasibility_batch(keep)
    assert_untouched(jm, engine, log_cap, call)


@pytest.mark.parametrize("engine, log_cap", CONFIGS, ids=CONFIG_IDS)
def test_conflict_batch_leaves_the_caller_tab(engine, log_cap):
    p = O.Problem(MIP)
    rng = np.random.default_rng(2)
    n, H = 24, p.M.shape[0]
    keep = (rng.random((n, H)) < 0.8).astype(np.uint8)  # the oracle's tableau is the tab's
    int_keep = (rng.random((n, len(p.ints))) < 0.7).astype(np.uint8)
    cuts = [[(int(rng.integers(0, 2)), int(rng.choice(p.ints)), float(rng.integers(0, 4)))
             for _ in range(int(rng.integers(0, 4)))] for _ in range(n)]
    cuts[3] = [(1, p.ints[0], 5.0)] * TALL_CUTS
    assert_untouched(MIP, engine, log_cap, lambda g: g.conflict_batch(keep, int_keep, cuts))


@pytest.mark.parametrize("engine, log_cap", CONFIGS, ids=CONFIG_IDS)
def test_column_batch_leaves_the_caller_tab(engine, log_cap):
    # every set has the snapshot's height: all resident or none, and the log cap sends sets to the redo
    p = O.Problem(MIP)
    keep = (np.random.default_rng(3).random((24, p.M.shape[1])) < 0.7).astype(np.uint8)
    keep[0] = 1
    assert_untouched(MIP, engine, log_cap, lambda g: g.column_batch(keep))


@pytest.mark.parametrize("engine, log_cap", CONFIGS, ids=CONFIG_IDS)
def test_scenario_batch_leaves_the_caller_tab(engine, log_cap):
    # the scenarios start from the caller's solved tableau, which they leave as it was, the snapshot included
    p = O.Problem(MIP)
    rng = np.random.default_rng(4)
    rows, cols = [int(v) for v in p.vrow[1:]], [int(v) for v in p.vcol[1:]]
    edits, offsets = [], [0]
    for _ in range(24):
        edits += [(0, int(rng.choice(rows)), float(rng.uniform(-20, 20))) for _ in range(int(rng.integers(0, 3)))]
        edits += [(1, int(rng.choice(cols)), float(rng.uniform(-5, 5))) for _ in range(int(rng.integers(0, 3)))]
        offsets.append(len(edits))
    assert_untouched(MIP, engine, log_cap, lambda g: g.scenario_batch(edits, offsets, check_cycles=True),
                     over_snapshot=False)


def _cuts(p, rng) -> list:
    return [(int(rng.integers(0, 2)), int(rng.choice(p.ints)), float(rng.integers(0, 4)))
            for _ in range(int(rng.integers(0, 4)))]


@pytest.mark.parametrize("engine, log_cap", CONFIGS, ids=CONFIG_IDS)
def test_pool_batch_leaves_the_caller_tab(engine, log_cap):
    p = O.Problem(MIP)
    col_of = {int(p.vcol[c]): c for c in range(1, len(p.vcol))}
    rng = np.random.default_rng(5)
    regions = [([(col_of[int(l)], float(rng.integers(0, 3))) for l in rng.choice(p.ints, int(rng.integers(0, 4)),
                                                                                replace=False)], _cuts(p, rng))
               for _ in range(24)]
    regions[3] = ([], [(1, p.ints[0], 5.0)] * TALL_CUTS)
    assert_untouched(MIP, engine, log_cap, lambda g: g.pool_batch(regions, check_cycles=True))


@pytest.mark.parametrize("engine, log_cap", CONFIGS, ids=CONFIG_IDS)
def test_target_batch_leaves_the_caller_tab(engine, log_cap):
    p = O.Problem(MIP)
    rng = np.random.default_rng(6)
    nodes = [([(1, int(rng.choice(p.ints)), float(rng.uniform(-5, 5))) for _ in range(int(rng.integers(0, 3)))],
              _cuts(p, rng)) for _ in range(24)]
    nodes[3] = ([(1, p.ints[1], 2.0)], [(1, p.ints[0], 5.0)] * TALL_CUTS)
    assert_untouched(MIP, engine, log_cap, lambda g: g.target_batch(nodes, check_cycles=True))


# ---- argument refusals ----------------------------------------------------------------------------------------------
def _i32(*v):
    return np.ascontiguousarray(v, dtype=np.int32)


def _refused(rc: int, code: int, msg: str):
    assert rc == code and _lib.load().jslp_last_error().decode() == msg, (rc, _lib.load().jslp_last_error(), msg)


INVALID = -1  # JSLP_E_INVALID


class _Out:
    """Output arrays for n sets of row_stride rows; `p(name)` is an array's address."""

    def __init__(self, n: int, row_stride: int):
        self.a = {k: np.zeros(n, dtype=np.int32) for k in ("status", "integral", "bvar", "pivots", "p1", "p2")}
        self.a.update({k: np.zeros(n, dtype=np.float64) for k in ("eval", "bval")})
        self.a["rhs"] = np.zeros((n, row_stride), dtype=np.float64)
        self.a["vrow"] = np.zeros((n, row_stride), dtype=np.int32)

    def p(self, name):
        return self.a[name].ctypes.data


def test_feasibility_and_column_batch_refusals():
    L = _lib.load()
    g, bare = _tab(MIP), _tab(MIP, save=False)
    H, W = g.height, g.width
    keep, out = np.ones((1, max(H, W)), dtype=np.uint8), _Out(1, H)
    try:
        _refused(L.jslp_feasibility_batch(None, keep.ctypes.data, 1, out.p("status"), None), INVALID, "tab is NULL")
        _refused(L.jslp_feasibility_batch(g.handle, None, 1, out.p("status"), None), INVALID,
                 "bad keep / verdict arguments")
        _refused(L.jslp_feasibility_batch(g.handle, keep.ctypes.data, -1, out.p("status"), None), INVALID,
                 "bad keep / verdict arguments")
        _refused(L.jslp_feasibility_batch(bare.handle, keep.ctypes.data, 1, out.p("status"), None), INVALID,
                 "feasibility_batch needs a snapshot (jslp_save)")
        _refused(L.jslp_column_batch(None, keep.ctypes.data, 1, out.p("status"), out.p("eval"), out.p("pivots"),
                                     out.p("rhs"), out.p("vrow")), INVALID, "tab is NULL")
        _refused(L.jslp_column_batch(g.handle, keep.ctypes.data, 1, out.p("status"), out.p("eval"), out.p("pivots"),
                                     out.p("rhs"), None), INVALID, "column_batch: bad keep / output arguments")
        _refused(L.jslp_column_batch(bare.handle, keep.ctypes.data, 1, out.p("status"), out.p("eval"),
                                     out.p("pivots"), out.p("rhs"), out.p("vrow")), INVALID,
                 "column_batch needs a snapshot (jslp_save)")
    finally:
        g.close()
        bare.close()


def test_scenario_batch_refusals():
    L = _lib.load()
    g = _tab(MIP)
    p = O.Problem(MIP)
    row, col = int(p.vrow[1]), int(p.vcol[1])
    out = _Out(2, g.height)

    def call(edits, offsets, n=None, tab=g, rhs=True):
        arr = (_lib.ScenarioEdit * max(1, len(edits or [])))()
        for i, (kind, index, d) in enumerate(edits or []):
            arr[i].kind, arr[i].index, arr[i].difference = kind, index, d
        n = len(offsets) - 1 if n is None else n
        return L.jslp_scenario_batch(tab.handle if tab is not None else None, arr if edits is not None else None,
                                     offsets.ctypes.data, n, 1, out.p("status"), out.p("eval"), out.p("p1"),
                                     out.p("p2"), out.p("rhs") if rhs else None, out.p("vrow"))

    try:
        _refused(call([], _i32(0, 0), tab=None), INVALID, "tab is NULL")
        _refused(call([], _i32(0, 0), rhs=False), INVALID, "scenario_batch: bad offsets / output arguments")
        _refused(call([(0, row, 1.0)], _i32(1, 1)), INVALID, "scenario_batch: offsets[0] must be 0")
        _refused(call([(0, row, 1.0)], _i32(0, 1, 0)), INVALID, "scenario_batch: offsets must not decrease")
        _refused(call(None, _i32(0, 1)), INVALID, "scenario_batch: edits is NULL")
        _refused(call([(2, row, 1.0)], _i32(0, 1)), INVALID,
                 "scenario_batch: edit kind must be 0 (rhs) or 1 (cost)")
        _refused(call([(1, col, 1.0), (0, row, 1.0)], _i32(0, 2)), INVALID,
                 "scenario_batch: a scenario's right-hand-side edits come before its cost edits")
        _refused(call([(0, 10 ** 6, 1.0)], _i32(0, 1)), INVALID,
                 "scenario_batch: unknown constraint or variable index")
    finally:
        g.close()


@pytest.mark.parametrize("entry", ["pool", "target"])
def test_pool_and_target_batch_refusals(entry):
    L = _lib.load()
    g, bare = _tab(MIP), _tab(MIP, save=False)
    p = O.Problem(MIP)
    lab = int(p.ints[0])
    fn = L.jslp_pool_batch if entry == "pool" else L.jslp_target_batch
    what, node = f"{entry}_batch", "region" if entry == "pool" else "node"
    stride = g.height + 2
    out = _Out(2, stride)

    def edit_array(items):
        if entry == "pool":
            arr = (_lib.Fix * max(1, len(items)))()
            for i, (c, v) in enumerate(items):
                arr[i].column, arr[i].value = c, v
        else:
            arr = (_lib.ScenarioEdit * max(1, len(items)))()
            for i, (kind, index, d) in enumerate(items):
                arr[i].kind, arr[i].index, arr[i].difference = kind, index, d
        return arr

    good = [(1, 1.0)] if entry == "pool" else [(1, lab, 1.0)]  # column 1 fixed at 1, or a cost edit

    def call(edits=good, edit_off=(0, 1), cuts=((1, lab, 2.0),), cut_off=(0, 1), tab=g, row_stride=stride,
             outputs=True, null_edits=False, null_cuts=False):
        n = len(edit_off) - 1
        carr = (_lib.Cut * max(1, len(cuts)))()
        for i, (ty, vi, val) in enumerate(cuts):
            carr[i].type, carr[i].var_index, carr[i].value = ty, vi, val
        eo, co = _i32(*edit_off), _i32(*cut_off)
        return fn(tab.handle if tab is not None else None, None if null_edits else edit_array(edits), eo.ctypes.data,
                  None if null_cuts else carr, co.ctypes.data, n, 1, row_stride, out.p("status"), out.p("eval"),
                  out.p("integral"), out.p("bvar"), out.p("bval"), out.p("pivots"), out.p("rhs"),
                  out.p("vrow") if outputs else None)

    try:
        assert call() == 0, _lib.load().jslp_last_error()
        _refused(call(tab=None), INVALID, "tab is NULL")
        _refused(call(outputs=False), INVALID, f"{what}: bad offsets / output arguments")
        _refused(call(tab=bare), INVALID, f"{what} needs a snapshot (jslp_save)")
        _refused(call(edit_off=(1, 1)), INVALID, f"{what}: offsets[0] must be 0")
        _refused(call(cut_off=(1, 1)), INVALID, f"{what}: offsets[0] must be 0")
        _refused(call(edit_off=(0, 1, 0), cut_off=(0, 0, 1)), INVALID, f"{what}: offsets must not decrease")
        _refused(call(edit_off=(0, 0, 1), cut_off=(0, 1, 0)), INVALID, f"{what}: offsets must not decrease")
        _refused(call(row_stride=g.height), INVALID,
                 f"{what}: row_stride is below a {node}'s height (rows plus cuts)")
        nulls = "fixes / cuts is NULL" if entry == "pool" else "edits / cuts is NULL"
        _refused(call(null_edits=True), INVALID, f"{what}: {nulls}")
        _refused(call(null_cuts=True), INVALID, f"{what}: {nulls}")
        if entry == "pool":
            _refused(call(edits=[(0, 1.0)]), INVALID, "pool_batch: fixed column out of range")
            _refused(call(edits=[(g.width, 1.0)]), INVALID, "pool_batch: fixed column out of range")
        else:
            _refused(call(edits=[(0, lab, 1.0)]), INVALID, "target_batch: edit kind must be 1 (cost)")
            _refused(call(edits=[(1, 10 ** 6, 1.0)]), INVALID, "target_batch: unknown variable index")
        cut_msg = f"{what}: cut type must be 0 (min) or 1 (max), on a label of the snapshot"
        _refused(call(cuts=((2, lab, 1.0),)), INVALID, cut_msg)
        _refused(call(cuts=((0, -1, 1.0),)), INVALID, cut_msg)
        _refused(call(cuts=((0, g.nVars, 1.0),)), INVALID, cut_msg)
    finally:
        g.close()
        bare.close()


def test_conflict_batch_refusals():
    L = _lib.load()
    g, bare = _tab(MIP), _tab(MIP, save=False)
    p = O.Problem(MIP)
    H, lab = g.height, int(p.ints[0])
    out = _Out(2, H + 2)
    keep = np.ones((2, H), dtype=np.uint8)
    int_keep = np.ones((2, len(p.ints)), dtype=np.uint8)

    def call(cut_off=(0, 1), cuts=((1, lab, 2.0),), tab=g, row_stride=H + 2, with_int_keep=True, null_cuts=False):
        n = len(cut_off) - 1
        carr = (_lib.Cut * max(1, len(cuts)))()
        for i, (ty, vi, val) in enumerate(cuts):
            carr[i].type, carr[i].var_index, carr[i].value = ty, vi, val
        co = _i32(*cut_off)
        return L.jslp_conflict_batch(tab.handle if tab is not None else None, keep.ctypes.data,
                                     int_keep.ctypes.data if with_int_keep else None, None if null_cuts else carr,
                                     co.ctypes.data, n, row_stride, out.p("status"), out.p("integral"), out.p("bvar"),
                                     out.p("bval"), out.p("pivots"), out.p("rhs"), out.p("vrow"))

    try:
        assert call() == 0, _lib.load().jslp_last_error()
        _refused(call(tab=None), INVALID, "tab is NULL")
        _refused(call(with_int_keep=False), INVALID, "conflict_batch: bad keep / offsets / output arguments")
        _refused(call(tab=bare), INVALID, "conflict_batch needs a snapshot (jslp_save)")
        _refused(call(cut_off=(1, 1)), INVALID, "conflict_batch: cut_offsets[0] must be 0")
        _refused(call(cut_off=(0, 1, 0)), INVALID, "conflict_batch: offsets must not decrease")
        _refused(call(row_stride=H), INVALID,
                 "conflict_batch: row_stride is below a node's height (kept rows plus cuts)")
        _refused(call(null_cuts=True), INVALID, "conflict_batch: cuts is NULL")
        _refused(call(cuts=((2, lab, 1.0),)), INVALID,
                 "conflict_batch: cut type must be 0 (min) or 1 (max), on a label of the snapshot")
    finally:
        g.close()
        bare.close()

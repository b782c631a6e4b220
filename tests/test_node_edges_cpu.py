"""CPU checks behind test_gpu_node_edges.py: its node-kernel shapes against the geometry an H100 SXM gives, the
half-integer MIP builder against the JSON front end and an independent solver, and the oracle's isIntegral /
getMostFractionalVar on the crafted tableaux against a few lines restating mip-utils.ts:43-61,100-126."""
import math

import numpy as np
import pytest

from test_gpu_node_edges import (K2_CASES, MIP_SCAN_CASES, NODE_LOG_HEAD, NODE_THREADS, NODE_WARPS, PREC,
                                 PRICE_BATCH, TIE_SMALL, U_BLOCK, D_SPLIT, mip_scan_tableau)
from test_gpu_shape_edges import H100_SXM, resident_rows, tie_arrays


def _bits(x):
    return np.float64(x).view(np.uint64)


def test_node_kernel_shapes_cross_every_edge():
    """Every shape fits the node kernel's shared memory on an H100 SXM (227 KB per block less 4 KB), and each split of
    the kernel is crossed from both sides: lanes (32 | 33 rows and columns), the D pass (128 | 129 rows), the ratio
    test's second pass per thread (256 | 257 rows), the U block (128 | 129 columns) and 50 | 51 priced columns."""
    dev = H100_SXM
    assert (NODE_THREADS, NODE_WARPS, D_SPLIT, U_BLOCK, PRICE_BATCH, NODE_LOG_HEAD) == (256, 8, 128, 128, 50, 64)
    assert resident_rows(dev, 33) == 748 and resident_rows(dev, 257) == 106
    shapes = [(resident_rows(dev, W) if H == "resident" else H, W) for _, H, W, _, _ in K2_CASES]
    assert all(H <= resident_rows(dev, W) for H, W in shapes)
    Hs, Ws = {H for H, _ in shapes}, {W for _, W in shapes}
    for below, above in ((32, 33), (D_SPLIT, D_SPLIT + 1), (NODE_THREADS, NODE_THREADS + 1)):
        assert below in Hs and above in Hs, (below, above)
    for below, above in ((32, 33), (U_BLOCK, U_BLOCK + 1), (PRICE_BATCH + 1, PRICE_BATCH + 2)):
        assert below in Ws and above in Ws, (below, above)
    assert max(W for W in Ws) > 2 * U_BLOCK and max(H for H in Hs) > 2 * NODE_THREADS
    # the tie LP of the scenario and feasibility batches takes the automatic engine's node kernel (H x W <= 16 384)
    assert 161 * 100 <= 16384 and 161 <= resident_rows(dev, 100)


def test_tie_rows_and_columns_are_copies():
    """The K2 placement of tie_arrays: tableau rows 2..9 reappear 32 and 256 rows on, the top-cost column 50 and 32
    columns on."""
    _, _, _, row_offsets, col_offsets = TIE_SMALL
    A, b, c, lower = tie_arrays(288, 59, 9001, 1, NODE_THREADS, 20, (32, 256), (PRICE_BATCH, 32))
    for off in (32, 256):
        assert np.array_equal(A[1:9], A[1 + off:9 + off]) and np.array_equal(b[1:9], b[1 + off:9 + off])
    assert c[1] == c.max()
    for off in (PRICE_BATCH, 32):
        assert np.array_equal(A[:, 1], A[:, 1 + off]) and c[1 + off] == c[1]
    assert row_offsets == (32, 128) and col_offsets == (PRICE_BATCH, 32)


def test_half_tie_mip_builder():
    """half_tie_mip_model: the front end's root tableau has the documented shape and integer variables; the LP
    relaxation leaves basic integer variables at exactly k + 1/2; the oracle's uncapped branch-and-cut reaches the
    optimum of SciPy's milp (HiGHS)."""
    pytest.importorskip("scipy")
    from scipy.optimize import Bounds, LinearConstraint, milp
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    from oracle import ref_model
    for n, group in ((12, 4), (20, 8)):
        jm = problems.half_tie_mip_model(n, group, seed=n)
        m = Model().loadJson(jm)
        it = m.initial_tableau()
        assert it.matrix.shape == (n + math.ceil(n / group) + 1, n + 1)
        assert len(it.integerIndices) == n
        root = ref_model.OracleTableau(it.matrix, it.varIndexByRow, it.varIndexByCol, fast_cycles=True)
        root.simplex()
        vr = root.maps()[0]
        ints = set(int(v) for v in it.integerIndices)
        halves = [x for r, x in enumerate(root.matrix()[:, 0]) if r and int(vr[r]) in ints and x - math.floor(x) == 0.5]
        assert len(halves) >= n // 2, (n, len(halves))
        names = list(jm["variables"])
        rows = list(jm["constraints"])
        A = np.array([[jm["variables"][v].get(r, 0.0) for v in names] for r in rows])
        ub = np.array([jm["constraints"][r]["max"] for r in rows])
        cost = -np.array([jm["variables"][v]["value"] for v in names])
        res = milp(cost, constraints=LinearConstraint(A, -np.inf, ub), integrality=np.ones(len(names)),
                   bounds=Bounds(0, np.inf))
        assert res.status == 0
        ores = ref_model.Solve(jm, fast_cycles=True)
        assert ores["feasible"] and abs(ores["result"] - (-res.fun)) <= 1e-9 * max(1.0, abs(res.fun)), (ores, res.fun)


def js_round(x):
    """Math.round: the nearest integer, halves toward +inf (x - floor(x) is exact)."""
    if x != x or math.isinf(x):
        return x
    f = math.floor(x)
    return float(f + 1) if x - f >= 0.5 else float(f)


def mip_utils(M, vrow, ints, precision=PREC):
    """isIntegral and getMostFractionalVar (mip-utils.ts:43-61, 100-126) over column 0 of M."""
    row_of = {int(v): r for r, v in enumerate(vrow) if r > 0}
    integral, biggest, sel, sel_val = True, 0.0, -1, 0.0
    for v in ints:
        r = row_of.get(int(v), -1)
        if r == -1:
            continue
        x = float(M[r, 0])
        fraction = abs(x - js_round(x))
        if fraction > precision:
            integral = False
        if fraction > biggest:
            biggest, sel, sel_val = fraction, int(v), x
    return integral, sel, sel_val


@pytest.mark.parametrize("H,kind", MIP_SCAN_CASES, ids=[f"H{h}-{k}" for h, k in MIP_SCAN_CASES])
def test_crafted_mip_scan_oracle_matches_mip_utils(H, kind):
    from test_gpu_lp_parity import oracle_lp
    it = mip_scan_tableau(H, kind, 100 + H)
    o = oracle_lp(it)
    integral, sel, val = mip_utils(it.matrix, it.varIndexByRow, it.integerIndices)
    iv, oval = o.most_fractional()
    assert o.is_integral() == integral
    assert iv == sel and _bits(oval) == _bits(val), (iv, oval, sel, val)
    if kind == "ties":   # many exact ties: the winner is the first tied entry of integerIndices, not the first row
        row_of = {int(v): r for r, v in enumerate(it.varIndexByRow) if r > 0}
        tied = [v for v in it.integerIndices if int(v) in row_of and abs(it.matrix[row_of[int(v)], 0]) % 1 == 0.5]
        assert sel == tied[0]

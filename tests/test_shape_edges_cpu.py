"""CPU checks behind the GPU shape-edge suite (test_gpu_shape_edges.py): its NumPy tableau builder is the front end's
tableau bit for bit, its geometry planner reproduces the thresholds the library states for an H100 SXM, and its tie and
threshold families are real LPs on which the oracle agrees with an independent solver."""
import numpy as np
import pytest

from helpers import highs_solve
from test_gpu_shape_edges import (H100_SXM, PP_MAX_ROWS, STEP_VARIANTS, THRESHOLDS, flat8_height, height_for,
                                  mixed_arrays, plan, resident_rows, threshold_arrays, tie_arrays)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("maximize", [True, False])
@pytest.mark.parametrize("family", ["mixed", "ties", "thresholds"])
def test_numpy_builder_equals_the_front_end(family, maximize):
    from jslpsolver_b200 import problems
    from jslpsolver_b200.model import Model
    if family == "mixed":
        A, b, c, lower = mixed_arrays(23, 17, 1, n_lower=5)
    elif family == "ties":
        A, b, c, lower = tie_arrays(60, 70, 2, 4, 4)
    else:
        A, b, c, lower = threshold_arrays(40, 30, 3)
    A[0, :len(THRESHOLDS)] = THRESHOLDS          # signed zeros and thresholds as explicit terms of a row
    c[-2:] = [-0.0, 0.0]                         # falsy costs
    assert lower.any() and not lower.all()
    want = Model().loadJson(problems.lp_model(A, b, c, lower, maximize)).initial_tableau()
    got = problems.lp_tableau(A, b, c, lower, maximize)
    assert np.array_equal(_bits(got.matrix), _bits(want.matrix))
    assert np.array_equal(got.varIndexByRow, want.varIndexByRow) and np.array_equal(got.varIndexByCol, want.varIndexByCol)
    assert np.array_equal(got.unrestricted, want.unrestricted) and got.optionalCosts.shape == want.optionalCosts.shape


def test_planner_reproduces_the_stated_thresholds():
    """132 SMs, 50 MB of L2: the ping-pong step runs up to H = 32 x 262 - 1 rows with the default variant and up to
    32 x 130 - 1 with 512 threads and one CTA per SM; the automatic variant turns to flat-8 once 16 rowcap stride bytes
    exceed 0.95 x L2; the shared-memory node kernel takes what fits 227 KB less 4 KB."""
    dev = H100_SXM
    for variant, G in ((10, 262), (3, 130), (9, 130)):
        assert height_for(dev, variant, PP_MAX_ROWS) == 32 * G - 1
        last, first = plan(dev, 32 * G - 1, 17, variant), plan(dev, 32 * G, 17, variant)
        assert last.pp and last.rows == 32 and last.G == G
        assert not first.pp and first.G == G + 2
    p = plan(dev, 8383, 17)
    assert (p.variant, p.grid, p.G, p.rows, p.pp) == (10, 264, 262, 32, True)
    # in-place look-ahead tail of the 128-thread variant at one CTA per SM: 16 895 rows fit, 16 896 do not
    assert plan(dev, 16895, 17, 5, grid_per_sm=1).rows_fit and not plan(dev, 16896, 17, 5, grid_per_sm=1).rows_fit
    H = flat8_height(dev, 400)
    assert 16.0 * (H + 64) * 400 > 0.95 * (50 << 20) >= 16.0 * (H + 63) * 400
    assert plan(dev, H, 400).variant == 11 and plan(dev, H - 1, 400).variant == 10 and plan(dev, H, 400).pp
    # a tall tableau past the threshold that the ping-pong step cannot take runs the in-place step
    assert not plan(dev, 9000, 400).pp and plan(dev, 9000, 400).variant == 11
    # co-residency of two ping-pong CTAs with a staged pivot row
    assert plan(dev, 108, 12000).pp and not plan(dev, 108, 16000).pp and plan(dev, 20, 25600).pp
    assert plan(dev, 108, 16000).coresident is False and plan(dev, 108, 25600).grid > dev.sms
    # resident node kernel: 176 H + 380 bytes at W = 17
    assert resident_rows(dev, 17) == (232448 - 4096 - 380) // 176
    assert len(STEP_VARIANTS) == 14


def _oracle(A, b, c, lower):
    from jslpsolver_b200 import problems
    from test_gpu_lp_parity import oracle_lp
    it = problems.lp_tableau(A, b, c, lower)
    o = oracle_lp(it)
    o.simplex()
    return o.state()


@pytest.mark.parametrize("family", ["ties", "thresholds"])
def test_families_agree_with_highs(family):
    """Same verdict and objective within 1e-7 relative as SciPy's HiGHS; some instances need phase 1 and are feasible
    and bounded.  An instance on which the oracle stops at a cycle has no verdict and is not counted."""
    pytest.importorskip("scipy")
    from jslpsolver_b200 import problems
    real = 0
    for seed in range(8):
        n_rows, n_vars = 30 + 7 * seed, 12 + 9 * seed
        if family == "ties":
            A, b, c, lower = tie_arrays(n_rows, n_vars, seed, 3, 4)
        else:
            A, b, c, lower = threshold_arrays(n_rows, n_vars, seed, extreme=False)
        st = _oracle(A, b, c, lower)
        if st.cyclePhase:
            continue   # the reference's rules stop on a cycle (degenerate ties can cycle): no verdict to compare
        status, val = highs_solve(problems.lp_model(A, b, c, lower))
        assert status in (0, 2, 3), (seed, status)
        assert bool(st.feasible) == (status != 2), (seed, status)
        if status == 0:
            ev = -st.evaluation   # the tableau minimises: a maximisation's optimum is the negated evaluation
            # threshold right-hand sides pin the optimum within HiGHS's 1e-7 feasibility tolerance of 0: absolute slack
            slack = 1e-6 if family == "thresholds" else 0.0
            assert st.bounded and abs(ev - val) <= 1e-7 * max(1.0, abs(val)) + slack, (seed, ev, val)
            real += st.lastP1 > 0
        elif status == 3:
            assert not st.bounded, seed
    assert real >= 3, real

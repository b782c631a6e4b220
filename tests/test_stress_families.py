"""The reference's stress families (src/solver.stress.test.ts:41-215: random LP / MIP, resource allocation,
transportation, single knapsack, set cover at 10..50 variables, seeded), restated with numpy generators
(jslpsolver_b200/problems.py).  The reference only asks its solver to finish with a verdict there; here

  * CPU: the oracle's verdict and optimum are compared with SciPy's HiGHS, which shares nothing with the reference;
  * GPU: Solve() on the CUDA path is compared with the oracle bit for bit -- result dict, node log, final tableau --
    for the default service at three speculation widths.
Multi-dimensional knapsacks (BASELINE config 5's family) small enough to terminate ride along.
"""
import numpy as np
import pytest

from helpers import highs_solve

SEEDS = (12345, 7, 99)   # 12345 is the seed the reference's suite uses


# BASELINE config 5's family (multi-dimensional 0/1 knapsack) at sizes whose branch-and-cut runs to termination with
# tolerance 0: 91 .. 1131 nodes in the oracle, optimum confirmed by HiGHS
MD_KNAPSACKS = ((20, 3, 1), (30, 5, 2), (40, 5, 3), (40, 8, 4), (60, 6, 5))


def suite():
    from jslpsolver_b200 import problems
    out = [(f"{label}-s{seed}", model) for seed in SEEDS for label, model in problems.stress_suite(seed)]
    out += [(f"md_knapsack_{n}x{m}-s{seed}", problems.knapsack_mip_model(n, m, seed)) for n, m, seed in MD_KNAPSACKS]
    return out


SUITE = suite()


def test_families_have_the_reference_shapes():
    """Sizes, names and row kinds of problem-generator.ts's families (a drifted generator would make the rest vacuous)."""
    from jslpsolver_b200 import problems
    m = problems.set_cover_model(15, 10, 1)
    assert m["opType"] == "min" and len(m["binaries"]) == 15 and all(c == {"min": 1.0} for c in m["constraints"].values())
    m = problems.transportation_model(4, 5, 1)
    assert len(m["variables"]) == 20 and sum("max" in c for c in m["constraints"].values()) == 4
    total = sum(c["max"] for c in m["constraints"].values() if "max" in c)
    assert all(c["min"] == total // 5 for c in m["constraints"].values() if "min" in c)
    m = problems.single_knapsack_model(20, 1)
    assert list(m["constraints"]) == ["capacity"] and len(m["binaries"]) == 20
    m = problems.random_mip_model(30, 15, 12345, 0.5, 0.3)
    assert 0 < len(m["ints"]) < 30 and set(m["ints"]) <= set(m["variables"])
    assert problems.random_lp_model(30, 15, 5) == problems.random_lp_model(30, 15, 5)   # solver.stress.test.ts:154-177
    assert len(problems.stress_suite()) == 18


@pytest.mark.parametrize("label,model", SUITE, ids=[s[0] for s in SUITE])
def test_oracle_agrees_with_an_independent_solver(label, model):
    pytest.importorskip("scipy")
    from oracle import ref_model
    status, val = highs_solve(model)
    res = ref_model.Solve(model, fast_cycles=True)
    if status == 0:
        assert res["feasible"] and res["bounded"], (label, res)
        assert abs(res["result"] - val) <= 1e-7 * max(1.0, abs(val)), (label, res["result"], val)
    elif status == 2:
        assert not res["feasible"], (label, res)
    else:
        # 3 = unbounded, 4 = HiGHS's presolve "unbounded or infeasible": either way no bounded optimum
        assert status in (3, 4) and not (res["feasible"] and res["bounded"]), (label, status, res)


@pytest.mark.gpu
@pytest.mark.parametrize("spec", [1, 8, 32, "hbm_slots"])
@pytest.mark.parametrize("label,model", SUITE, ids=[s[0] for s in SUITE])
def test_gpu_matches_oracle_bit_for_bit(label, model, spec):
    import jslpsolver_b200 as J
    from oracle import ref_model
    from test_gpu_lp_parity import same_bits
    is_mip = bool(model.get("ints") or model.get("binaries"))
    if not is_mip and spec != 1:
        pytest.skip("speculation width only matters with integer variables")
    if spec == "hbm_slots" and not label.startswith("md_knapsack"):
        pytest.skip("HBM node slots: exercised on the trees that are deep enough to fill them")
    osol = ref_model.solve_full(model, fast_cycles=True, node_log=1 << 16)
    s = J.Solver()
    if spec == "hbm_slots":   # K3: 3 node slots of 5-step graphs over HBM-resident nodes, 16 speculated per round
        s.engine, s.max_spec_batch, s.node_slots, s.slot_steps = 2, 16, 3, 5
    else:
        s.max_spec_batch = spec
    gsol = s.Solve(model, full=True)
    ores = ref_model.Solve(model, fast_cycles=True)
    gres = J.Solve(model)
    assert list(gres.keys()) == list(ores.keys()), (label, gres, ores)
    for k in ores:
        assert gres[k] == ores[k] or (gres[k] != gres[k] and ores[k] != ores[k]), (label, k, gres[k], ores[k])
    gt = gsol._tableau
    if osol.tableau is None:
        return
    st = osol.state
    assert (gt.feasible, gt.bounded) == (bool(st.feasible), bool(st.bounded)), label
    assert same_bits(gt.matrix2d(), osol.tableau.matrix()), label
    assert np.array_equal(gt.varIndexByRow, osol.tableau.maps()[0]) and np.array_equal(gt.varIndexByCol, osol.tableau.maps()[1])
    if is_mip:
        onl, gnl = osol.tableau.node_log(), gt.node_log()
        assert gnl.shape == onl.shape, (label, gnl.shape, onl.shape)
        for i in range(len(onl)):
            a, b = gnl[i], onl[i]
            ok = all(a[k] == b[k] for k in (0, 1, 2, 4, 5, 7)) and same_bits(a[6], b[6]) and (not b[2] or same_bits(a[3], b[3]))
            assert ok, f"{label} node {i}: gpu={a.tolist()} oracle={b.tolist()}"
        assert gt.branchAndCutIterations == st.bncIterations

"""CPU checks of the irreducible infeasible subset (DESIGN.md section 2c): the oracle's literal deletion filter gives
sets that SciPy's HiGHS finds infeasible with every one-row-smaller subset feasible (golden fixtures, random LPs,
planted conflicts), the production schedule `deletion_filter` driven by the oracle's test equals the literal filter
at every width, the certificate start set is infeasible, the ValueError cases and the C prototype."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_bundle
from helpers import strip_timeouts

BUNDLE = load_bundle()
INFEASIBLE_FIXTURES = [f for f in BUNDLE["fixtures"] if f.get("expects", {}).get("feasible") is False
                       and not (f["model"].get("ints") or f["model"].get("binaries"))]


def _model(jm):
    from jslpsolver_b200.model import Model
    return Model().loadJson(strip_timeouts(jm))


def _highs_feasible(it, rows):
    """Is {x : A x <= b over `rows` of the initial tableau, x >= 0 unless unrestricted} non-empty?  Row r of the
    initial tableau reads slack_r = M[r,0] - M[r,1:] x >= 0."""
    from scipy.optimize import linprog
    M = it.matrix
    n = M.shape[1] - 1
    if not rows:
        return True
    bounds = [(None, None) if it.unrestricted[it.varIndexByCol[c]] else (0, None) for c in range(1, n + 1)]
    res = linprog(np.zeros(n), A_ub=M[rows, 1:], b_ub=M[rows, 0], bounds=bounds, method="highs")
    assert res.status in (0, 2), res.message
    return res.status == 0


def _assert_irreducible_by_highs(it, rows):
    assert not _highs_feasible(it, rows), f"{rows} is feasible under HiGHS"
    for s in rows:
        assert _highs_feasible(it, [r for r in rows if r != s]), f"{rows} minus {s} is still infeasible under HiGHS"


def _describe(m, rows):
    return [{"name": m.constraints[r - 1].name if m.constraints[r - 1].name is not None else m.constraints[r - 1].index,
             "type": "max" if m.constraints[r - 1].isUpperBound else "min", "rhs": m.constraints[r - 1].rhs} for r in rows]


@pytest.mark.parametrize("fx", INFEASIBLE_FIXTURES, ids=lambda f: f["file"])
def test_fixture_literal_filter_is_an_iis(fx):
    from oracle import iis as O
    m = _model(fx["model"])
    it = m.initial_tableau()
    res = O.iis(it, m.precision)
    if fx["file"] == "ChenhuaWANG22_2.json":
        # phase 1 of the whole LP cycles: its test is undecided, so iis() refuses it.  The literal filter over every
        # row still ends on a set it proved infeasible, with rows kept on undecided verdicts.
        assert res is None
        rows = list(range(1, it.matrix.shape[0]))
        assert O.test(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, m.precision, rows)[0] == O.UNDECIDED
        kept, irreducible = O.literal_filter(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted,
                                             m.precision, rows)
        assert not irreducible and not _highs_feasible(it, kept)
        return
    kept, irreducible, _ = res
    assert irreducible
    _assert_irreducible_by_highs(it, kept)


def test_infeasible_berlin_airlift():
    """The `brit` row shares its name with a variable and no variable has a coefficient in it: it reads 0 >= 13."""
    from oracle import iis as O
    fx = [f for f in INFEASIBLE_FIXTURES if f["file"] == "Infeasible Berlin Air Lift Problem.json"][0]
    m = _model(fx["model"])
    kept, irreducible, _ = O.iis(m.initial_tableau(), m.precision)
    assert _describe(m, kept) == [{"name": "brit", "type": "min", "rhs": 13}] and irreducible


def _random_infeasible(n_seeds=50):
    from jslpsolver_b200 import problems
    out = []
    seed = 0
    while len(out) < n_seeds and seed < 2000:
        rng = np.random.default_rng(seed)
        n, mcons = int(rng.integers(4, 41)), int(rng.integers(3, 31))
        jm = problems.random_lp_model(n, mcons, seed=1000 + seed)
        m = _model(jm)
        it = m.initial_tableau()
        if not _highs_feasible(it, list(range(1, it.matrix.shape[0]))):
            out.append((seed, m, it))
        seed += 1
    return out


RANDOM = None


def _random():
    global RANDOM
    if RANDOM is None:
        RANDOM = _random_infeasible()
    return RANDOM


def test_random_lps_literal_filter_is_an_iis():
    from oracle import iis as O
    cases = _random()
    undecided = 0
    for seed, m, it in cases:
        res = O.iis(it, m.precision)
        if res is None:  # HiGHS says infeasible; phase 1 may only cycle, never call it feasible
            rows = list(range(1, it.matrix.shape[0]))
            assert O.test(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, m.precision,
                          rows)[0] == O.UNDECIDED, seed
            undecided += 1
            continue
        kept, irreducible, _ = res
        assert irreducible, seed
        _assert_irreducible_by_highs(it, kept)
    print(f"{len(cases)} infeasible random LPs, {undecided} with a cycling phase 1")
    assert len(cases) - undecided >= 40


@pytest.mark.parametrize("n_vars,n_cons,k,seed", [(12, 10, 2, 1), (20, 15, 4, 2), (40, 30, 6, 3), (60, 40, 9, 4)])
def test_planted_models(n_vars, n_cons, k, seed):
    from jslpsolver_b200 import problems
    from oracle import iis as O
    jm = problems.planted_infeasible_model(n_vars, n_cons, k, seed)
    m = _model(jm)
    it = m.initial_tableau()
    kept, irreducible, _ = O.iis(it, m.precision)
    assert irreducible
    assert sorted(c["name"] for c in _describe(m, kept)) == sorted(f"conflict{p}" for p in range(k))
    _assert_irreducible_by_highs(it, kept)


def _oracle_batch(it, precision, counter):
    from oracle import iis as O

    def test_batch(sets):
        counter[0] += len(sets)
        return [O.test(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, precision, s)[0] for s in sets]
    return test_batch


def test_schedule_equals_the_literal_filter():
    """The production schedule, driven by the oracle's test, commits exactly the literal filter's decisions at every
    width, with and without the pre-pass."""
    from jslpsolver_b200 import problems
    from jslpsolver_b200.iis import deletion_filter
    from oracle import iis as O
    cases = [(m, m.initial_tableau()) for m in (_model(f["model"]) for f in INFEASIBLE_FIXTURES)]
    cases += [(m, it) for _, m, it in _random()[:15]]
    for k, seed in ((3, 5), (7, 6)):
        m = _model(problems.planted_infeasible_model(30, 24, k, seed))
        cases.append((m, m.initial_tableau()))
    for m, it in cases:
        rows = list(range(1, it.matrix.shape[0]))
        want = O.literal_filter(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, m.precision, rows)
        for width in (1, 2, 7, 64):
            for prepass in (False, True):
                n = [0]
                got = deletion_filter(_oracle_batch(it, m.precision, n), rows, width, prepass)
                assert got == want, (width, prepass)
                if width == 1:
                    assert n[0] == len(rows)  # the literal filter: one test per row


def test_schedule_with_scripted_verdicts():
    """A scripted test (infeasible iff the set contains rows 2 and 5, undecided when it lacks row 7) checks the commit
    rule, the undecided-keeps rule and `irreducible` without any LP."""
    from jslpsolver_b200.iis import INFEASIBLE, UNDECIDED, FEASIBLE, deletion_filter

    def verdict(s):
        if 7 not in s and 2 in s and 5 in s:
            return UNDECIDED
        return INFEASIBLE if 2 in s and 5 in s else FEASIBLE
    rows = list(range(1, 11))
    for width in (1, 2, 3, 10, 64):
        for prepass in (False, True):
            kept, irreducible = deletion_filter(lambda sets: [verdict(s) for s in sets], rows, width, prepass)
            assert kept == [2, 5, 7] and not irreducible


def test_certificate_start_set_is_infeasible():
    """Wherever S0 is the certificate support, HiGHS also finds it infeasible; the share of fallbacks to all rows is
    reported."""
    from jslpsolver_b200 import problems
    from oracle import iis as O
    cases = [(f["file"], _model(f["model"])) for f in INFEASIBLE_FIXTURES]
    cases += [(f"random seed {s}", m) for s, m, _ in _random()]
    cases += [(f"planted {k}", _model(problems.planted_infeasible_model(40, 30, k, k))) for k in (2, 5, 8)]
    fallback = undecided = 0
    for label, m in cases:
        it = m.initial_tableau()
        S0, support, _ = O.start_set(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted, m.precision)
        if S0 is None:  # the whole LP's phase 1 cycles: no certificate
            undecided += 1
            continue
        if S0 == support:
            assert not _highs_feasible(it, S0), label
        else:
            fallback += 1
    decided = len(cases) - undecided
    print(f"certificate support used on {decided - fallback} of {decided} models, all rows on {fallback}")
    assert fallback < decided


class _StubTableau:
    def __init__(self, model):
        self.model = model
        self.handle = None
        self._version = 0
        self._solved_version = -1
        self.context = None


def test_value_errors():
    from jslpsolver_b200.tableau import Solution
    bad = [f for f in INFEASIBLE_FIXTURES if f["file"] == "Infeasible Berlin Air Lift Problem.json"][0]["model"]
    lp = strip_timeouts([f for f in BUNDLE["fixtures"] if f["file"] == "Berlin Air Lift Problem.json"][0]["model"])
    cases = [
        (dict(bad, binaries={"brit": 1}), False, "integer or binary"),
        (dict(bad, ints={"brit": 1}), False, "integer or binary"),
        (dict(bad, constraints=dict(bad["constraints"], plane={"max": 44, "weight": 10})), False, "soft constraints"),
        (dict(bad, constraints=dict(bad["constraints"], plane={"max": 44, "priority": "strong"})), False, "soft constraints"),
        (lp, True, "feasible"),
    ]
    for jm, feasible, match in cases:
        t = _StubTableau(_model(jm))
        with pytest.raises(ValueError, match=match):
            Solution(t, 0.0, feasible, True).iis()
    t = _StubTableau(_model(bad))
    s = Solution(t, 0.0, False, True)
    t._version += 1
    with pytest.raises(ValueError, match="edited or solved again"):
        s.iis()
    t = _StubTableau(_model(bad))
    s = Solution(t, 0.0, False, True)
    t.handle, t._solved_version, t._version = object(), 3, 4
    s._version = 4
    with pytest.raises(ValueError, match="edited or solved again"):
        s.iis()
    with pytest.raises(ValueError, match="needs a solution of a Model"):
        Solution(_StubTableau(None), 0.0, False, True).iis()


def test_ctypes_signature_matches_the_header():
    from jslpsolver_b200 import _lib
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+jslp_feasibility_batch\s*\(([^)]*)\)\s*;", header)
    assert proto, "jslp_feasibility_batch is not declared"
    params = [p.strip() for p in proto.group(1).split(",")]
    types = [re.sub(r"\s+", " ", p.rsplit("*", 1)[0]).strip() + " *" if "*" in p else p.rsplit(" ", 1)[0] for p in params]
    assert types == ["jslp_tab *", "const uint8_t *", "int", "int32_t *", "int32_t *"], types
    (name, res, args), = [s for s in _lib.SYMBOLS if s[0] == "jslp_feasibility_batch"]
    C = _lib.C
    assert res is C.c_int and args == [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]

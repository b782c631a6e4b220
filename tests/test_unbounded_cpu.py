"""CPU checks of Solution.unbounded() (DESIGN.md section 2l): the oracle restatement's bounding set makes the LP bounded
under SciPy's HiGHS and every one-cap-smaller set leaves it unbounded (planted leaks, seeded random LPs, the unbounded
fixture), the planted models give the closed-form set, the ray is an exact improving certificate on integer models, a
stop that the ratio-test threshold made spurious is not confirmed, the production schedule equals the literal filter,
and the ValueError cases and the C prototypes."""
import os
import re
from fractions import Fraction

import numpy as np
import pytest

from conftest import ROOT, load_bundle
from helpers import strip_timeouts

import unbounded_oracle as UO

BUNDLE = load_bundle()
CYCLING = [f for f in BUNDLE["fixtures"] if f["file"] == "Cycling introductory example.json"][0]["model"]
EXAMPLE = {"optimize": "profit", "opType": "max",
           "constraints": {"c": {"max": 4}, "d": {"min": 1}},
           "variables": {"x": {"profit": 1, "c": 1, "d": 1}, "y": {"profit": 2, "c": -1}}}
SPURIOUS = {"optimize": "x", "opType": "max", "constraints": {"c": {"max": 5e-8}}, "variables": {"x": {"x": 1, "c": 10}}}
CAP = 1e6


def _model(jm):
    return UO.presolved_model(strip_timeouts(jm))


def _linprog_status(it, capped_labels):
    """HiGHS status of max M[0,1:].x over the initial tableau's rows, x >= 0, with x <= CAP on `capped_labels`."""
    from scipy.optimize import linprog
    M = it.matrix
    bounds = [(0, CAP if int(it.varIndexByCol[c]) in capped_labels else None) for c in range(1, M.shape[1])]
    res = linprog(-M[0, 1:], A_ub=M[1:, 1:] if M.shape[0] > 1 else None, b_ub=M[1:, 0] if M.shape[0] > 1 else None,
                  bounds=bounds, method="highs")
    assert res.status in (0, 2, 3), res.message
    return res.status


def _assert_irreducible_by_highs(m, ids):
    it = m.initial_tableau()
    label = {v.id: v.index for v in m.variables}
    caps = {label[i] for i in ids}
    assert _linprog_status(it, caps) == 0, f"caps on {ids} leave the LP unbounded under HiGHS"
    for s in ids:
        assert _linprog_status(it, caps - {label[s]}) == 3, f"{ids} minus {s} still bounds the LP under HiGHS"


def _closed_form(jm):
    return [v for v in jm["variables"] if v.startswith("solo") or v.startswith("pairV")]


PLANTED = [(30, 20, 3, 2, 1), (40, 30, 0, 3, 2), (25, 18, 4, 0, 3), (60, 45, 5, 4, 4), (14, 8, 1, 3, 5)]


@pytest.mark.parametrize("n_vars,n_cons,n_solo,n_pairs,seed", PLANTED)
def test_planted_models_give_the_closed_form_set(n_vars, n_cons, n_solo, n_pairs, seed):
    from jslpsolver_b200 import problems
    jm = problems.planted_unbounded_model(n_vars, n_cons, n_solo, n_pairs, seed)
    m = _model(jm)
    r = UO.unbounded(m)
    assert r is not None and r["confirmed"] is True and r["blocking"] == []
    assert r["bound"] == {"variables": _closed_form(jm), "irreducible": True}
    _assert_irreducible_by_highs(m, r["bound"]["variables"])


def _random_unbounded(limit=12):
    from jslpsolver_b200 import problems
    found = []
    for seed in range(400):
        jm = problems.random_lp_model(8, 6, seed=seed) if seed % 2 else problems.mixed_lp_model(8, 6, seed=seed)
        m = _model(jm)
        it = m.initial_tableau()
        F, vr, vc, st = UO.stop_tableau(it, m.precision)
        if st.feasible and not st.bounded and not st.cyclePhase:
            found.append((seed, jm))
        if len(found) >= limit:
            break
    return found


def test_random_unbounded_lps_against_highs():
    cases = _random_unbounded()
    assert len(cases) >= 6, "too few seeded models come out unbounded"
    for seed, jm in cases:
        m = _model(jm)
        r = UO.unbounded(m)
        if r["confirmed"]:
            assert r["bound"] is not None and r["bound"]["variables"], seed
            _assert_irreducible_by_highs(m, r["bound"]["variables"])
        else:  # the stop was a ratio-test artefact: HiGHS finds the LP bounded
            assert _linprog_status(m.initial_tableau(), set()) == 0, seed


def test_cycling_fixture():
    m = _model(CYCLING)
    r = UO.unbounded(m)
    assert r is not None
    if r["bound"] is not None and r["confirmed"]:
        _assert_irreducible_by_highs(m, r["bound"]["variables"])
    else:  # an undecided cone test must be reported, not hidden
        assert r["bound"] is None or r["bound"]["irreducible"] is False or r["confirmed"] is not True


def test_example_from_the_contract():
    r = UO.unbounded(_model(EXAMPLE))
    assert r["ray"] == {"y": 1.0} and r["rate"] == 2.0 and r["point"] == {"x": 1.0}
    assert [(c["name"], c["activity"], c["rate"]) for c in r["constraints"]] == [("c", 1.0, -1.0), ("d", 1.0, 0.0)]
    assert r["blocking"] == [] and r["confirmed"] is True
    assert r["bound"] == {"variables": ["y"], "irreducible": True}


def test_spurious_stop_is_not_confirmed():
    m = _model(SPURIOUS)
    it = m.initial_tableau()
    _, _, _, st = UO.stop_tableau(it, m.precision)
    assert st.feasible and not st.bounded  # the reference's ratio test skips the blocking row
    assert _linprog_status(it, set()) == 0  # HiGHS: x <= 5e-9
    r = UO.unbounded(m)
    assert r["confirmed"] is False and r["blocking"] == ["c"]
    assert r["bound"] == {"variables": [], "irreducible": True}


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_ray_is_an_exact_certificate_on_integer_models(seed):
    from jslpsolver_b200 import problems
    jm = problems.planted_unbounded_model(20, 14, 2, 2, seed)
    m = _model(jm)
    r = UO.unbounded(m)
    d = {k: Fraction(v) for k, v in r["ray"].items()}
    x = {k: Fraction(v) for k, v in r["point"].items()}
    obj = sum(Fraction(jm["variables"][k].get("profit", 0)) * v for k, v in d.items())
    assert obj > 0 and r["rate"] > 0 and Fraction(r["rate"]) == obj
    for row in r["constraints"]:
        a = {k: Fraction(v.get(row["name"], 0)) for k, v in jm["variables"].items()}
        rate = sum(a[k] * v for k, v in d.items())
        act = sum(a[k] * v for k, v in x.items())
        assert Fraction(row["rate"]) == rate, row
        assert abs(Fraction(row["activity"]) - act) <= Fraction(1, 10 ** 9) * (1 + abs(act)), row
        assert rate <= 0 if row["type"] == "max" else rate >= 0
    assert r["blocking"] == []


def _oracle_batch(K, vr, vc, P, cols):
    from jslpsolver_b200.unbounded import BOUNDED, RAY, UNDECIDED
    code = {UO.RAY: RAY, UO.BOUNDED: BOUNDED, UO.UNDECIDED: UNDECIDED}
    return lambda sets: [(code[v], s) for v, s in (UO.test(K, vr, vc, P, S, cols)[:2] for S in sets)]


def test_schedule_equals_the_literal_filter():
    """bounding_set, driven by the oracle's cone test, gives the literal filters' answer at every width."""
    from jslpsolver_b200 import problems
    from jslpsolver_b200.unbounded import bounding_set
    cases = [problems.planted_unbounded_model(*p) for p in PLANTED[:3]] + [jm for _, jm in _random_unbounded(5)]
    for jm in cases:
        m = _model(jm)
        it = m.initial_tableau()
        H, W = it.matrix.shape
        structural = {v.index for v in m.variables}
        cols = [c for c in range(1, W) if int(it.varIndexByCol[c]) in structural]
        K, vr, vc = UO.cone(it.matrix, it.varIndexByRow, it.varIndexByCol, W + H - 2)
        confirmed, B, irreducible, _ = UO.bound(K, vr, vc, m.precision, cols)
        for width in (1, 2, 5, 64):
            for prepass in (False, True):
                got = bounding_set(_oracle_batch(K, vr, vc, m.precision, cols), len(cols), width, prepass)
                assert got == (confirmed, B, irreducible), (jm.get("name"), width, prepass)


def test_schedule_with_scripted_verdicts():
    """A scripted cone test -- bounded iff columns 2 and 5 are capped, undecided once they are but 7 is not, and a
    ray's support the uncapped columns of {2, 5, 7} -- checks the additive phase, the mapped deletion filter and
    `irreducible` without any LP."""
    from jslpsolver_b200.unbounded import BOUNDED, RAY, UNDECIDED, bounding_set

    def verdict(S):
        if 2 in S and 5 in S:
            return (BOUNDED, []) if 7 in S else (UNDECIDED, [])
        return RAY, [c for c in (2, 5, 7) if c not in S]
    for width in (1, 2, 3, 10, 64):
        for prepass in (False, True):
            confirmed, kept, irreducible = bounding_set(lambda sets: [verdict(s) for s in sets], 10, width, prepass)
            assert confirmed is True and kept == [2, 5, 7] and not irreducible

    def verdict2(S):  # a clean case: bounded iff {3, 8} are capped; the rays name both at once
        return (BOUNDED, []) if {3, 8} <= set(S) else (RAY, [c for c in (1, 3, 8) if c not in S])
    for width in (1, 4):
        assert bounding_set(lambda sets: [verdict2(s) for s in sets], 10, width) == (True, [3, 8], True)
    assert bounding_set(lambda sets: [(UNDECIDED, [])] * len(sets), 10, 4) == (None, None, False)
    assert bounding_set(lambda sets: [(BOUNDED, [])] * len(sets), 10, 4) == (False, [], True)


class _StubTableau:
    def __init__(self, model):
        self.model = model
        self.handle = None
        self._version = 0
        self._solved_version = -1
        self.context = None


def test_value_errors():
    from jslpsolver_b200.tableau import Solution
    from jslpsolver_b200.model import Model
    lp = dict(EXAMPLE)
    cases = [
        (dict(lp, binaries={"x": 1}), True, False, "integer or binary"),
        (dict(lp, ints={"y": 1}), True, False, "integer or binary"),
        (dict(lp, constraints=dict(lp["constraints"], c={"max": 4, "weight": 10})), True, False, "soft constraints"),
        (dict(lp, constraints=dict(lp["constraints"], c={"max": 4, "priority": "strong"})), True, False,
         "soft constraints"),
        (dict(lp, unrestricted={"x": 1}), True, False, "unrestricted"),
        (lp, True, True, "bounded"),
        (lp, False, True, "infeasible"),
    ]
    for jm, feasible, bounded, match in cases:
        t = _StubTableau(Model().loadJson(jm))
        with pytest.raises(ValueError, match=match):
            Solution(t, 0.0, feasible, bounded).unbounded()
    t = _StubTableau(Model().loadJson(lp))
    s = Solution(t, 0.0, True, False)
    t._version += 1
    with pytest.raises(ValueError, match="edited or solved again"):
        s.unbounded()
    t = _StubTableau(Model().loadJson(lp))
    s = Solution(t, 0.0, True, False)
    t.handle, t._solved_version, t._version = object(), 3, 4
    s._version = 4
    with pytest.raises(ValueError, match="edited or solved again"):
        s.unbounded()
    with pytest.raises(ValueError, match="needs a solution of a Model"):
        Solution(_StubTableau(None), 0.0, True, False).unbounded()


def _types(name):
    header = open(os.path.join(ROOT, "include", "jslp_b200.h")).read()
    proto = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", header)
    assert proto, f"{name} is not declared"
    params = [p.strip() for p in proto.group(1).split(",")]
    return [re.sub(r"\s+", " ", p.rsplit("*", 1)[0]).strip() + " *" if "*" in p else p.rsplit(" ", 1)[0]
            for p in params]


def test_ctypes_signatures_match_the_header():
    from jslpsolver_b200 import _lib
    C, P = _lib.C, _lib.C.c_void_p
    want = {
        "jslp_cone_create": (["jslp_tab *", "jslp_tab * *"], [P, C.POINTER(P)]),
        "jslp_column_batch": (["jslp_tab *", "const uint8_t *", "int", "int32_t *", "double *", "int32_t *",
                               "double *", "int32_t *"], [P, P, C.c_int, P, P, P, P, P]),
        "jslp_column": (["jslp_tab *", "int", "double *"], [P, C.c_int, P]),
    }
    for name, (types, args) in want.items():
        assert _types(name) == types, (name, _types(name))
        (_, res, got), = [s for s in _lib.SYMBOLS if s[0] == name]
        assert res is C.c_int and got == args, name

"""The IIS feasibility test (DESIGN.md section 2c) and the MIP conflict's node LPs (section 2n) are one row-subset batch:
jslp_feasibility_batch equals jslp_conflict_batch with an empty integer mask and no cuts, set by set, on continuous
models and on a MIP tableau (where the feasibility test runs the node kernel without an integer mask), through the node
kernel and the single-tableau path.  A feasibility call asks for no column outputs, so every set that fits shared
memory runs in one launch however many there are; a set that keeps no row is decided without a launch."""
from __future__ import annotations

import numpy as np
import pytest

import conflict_oracle as O
from conftest import load_bundle
from helpers import strip_timeouts
from jslpsolver_b200 import _lib, problems

pytestmark = pytest.mark.gpu


def _gpu(jm: dict, engine=None):
    from jslpsolver_b200.model import Model
    from jslpsolver_b200.tableau import GpuTableau
    m = Model().loadJson(jm)
    g = GpuTableau(m.precision)
    g.setModel(m)
    if engine is not None:
        g.set_option(_lib.OPT_ENGINE, engine)
    g.save()
    return g


def _chenhua() -> dict:
    b = load_bundle()
    return strip_timeouts([f for f in b["fixtures"] if f["file"] == "ChenhuaWANG22_2.json"][0]["model"])


MODELS = {
    "ChenhuaWANG22_2": _chenhua,                                                    # continuous, cycling phase 1
    "mixed 40x30": lambda: problems.mixed_lp_model(40, 30, 11, frac_min=0.5),        # continuous
    "planted conflict 30x40": lambda: problems.planted_integer_conflict_model(30, 40, 4, 3),  # MIP
}


@pytest.mark.parametrize("engine", [None, 2], ids=["k2", "engine2"])
@pytest.mark.parametrize("name", list(MODELS))
def test_feasibility_equals_a_conflict_node_without_mask_or_cuts(name, engine):
    jm = MODELS[name]()
    p = O.Problem(jm)
    H = p.M.shape[0]
    keep = np.ones((H + 1, H), dtype=np.uint8)  # every row, no row, and every row but one
    keep[1] = 0
    for s in range(1, H):
        keep[s + 1, s] = 0
    rng = np.random.default_rng(5)
    keep = np.vstack([keep, (rng.random((12, H)) < 0.8).astype(np.uint8)])
    g = _gpu(jm, engine)
    verdict, pivots = g.feasibility_batch(keep)
    res = g.conflict_batch(keep, np.zeros((len(keep), len(p.ints)), dtype=np.uint8), [[] for _ in keep])
    g.close()
    assert verdict.tolist() == res["status"].tolist()
    assert pivots.tolist() == res["pivots"].tolist()
    assert (name == "planted conflict 30x40") == (len(p.ints) > 0)
    if name == "ChenhuaWANG22_2":
        assert (verdict == 2).sum() >= 10


def _tall_lp(rows: int, seed: int) -> dict:
    """2 variables and `rows` constraints, every tenth a lower bound: a tall, narrow LP whose phase 1 takes a few
    pivots."""
    rng = np.random.default_rng(seed)
    cons, x, y = {}, {"obj": 1.0}, {"obj": 1.0}
    for i in range(rows):
        cons[f"r{i}"] = {"min": float(rng.uniform(0.5, 1.0))} if i % 10 == 0 else {"max": float(rng.uniform(10, 20))}
        x[f"r{i}"], y[f"r{i}"] = float(rng.uniform(0.5, 2.0)), float(rng.uniform(0.5, 2.0))
    return {"optimize": "obj", "opType": "max", "constraints": cons, "variables": {"x": x, "y": y}}


def test_feasibility_sets_that_fit_run_in_one_launch():
    """1500 sets of a 2000-row LP with 2 variables all fit shared memory: one launch, although column outputs would
    bound a launch at 1397 sets as tall as the first (every row; about 32 MB of outputs), as the conflict batch's two
    launches show."""
    jm = _tall_lp(2000, 17)
    g = _gpu(jm)
    H = g.matrix2d().shape[0]
    assert H == 2001
    keep = (np.random.default_rng(3).random((1500, H)) < 0.9).astype(np.uint8)
    keep[0] = 1
    n0 = g.context.launches
    verdict, pivots = g.feasibility_batch(keep)
    n1 = g.context.launches
    res = g.conflict_batch(keep, np.zeros((len(keep), 0), dtype=np.uint8), [[] for _ in keep])
    n2 = g.context.launches
    g.close()
    assert n1 - n0 == 1
    assert n2 - n1 == 2
    assert verdict.tolist() == res["status"].tolist() and pivots.tolist() == res["pivots"].tolist()
    assert (pivots > 0).any()


def test_sets_without_rows_make_no_launch():
    g = _gpu(MODELS["mixed 40x30"](), engine=2)
    H = g.matrix2d().shape[0]
    n0 = g.context.launches
    none = g.feasibility_batch(np.zeros((0, H), dtype=np.uint8))
    verdict, pivots = g.feasibility_batch(np.zeros((3, H), dtype=np.uint8))
    assert g.context.launches == n0
    g.close()
    assert none[0].size == 0
    assert verdict.tolist() == [0, 0, 0] and pivots.tolist() == [0, 0, 0]

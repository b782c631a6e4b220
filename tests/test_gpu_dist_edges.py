"""Sharded branch and cut at 2, 3 and 4 ranks (tests/dist_edges_worker.py under torchrun, every rank on cuda:0 over gloo;
over NCCL with one GPU per rank when the box has them): every rank must commit identically, in the reference's order
(DESIGN.md section 5), on every evaluation path and stop rule, with optional objectives on the wire.

Every case checks (a) identical ranks: every status field but the per-rank work counters, the node log, the final
tableau and labels, the result and model.solutions, bit for bit; (b) parity with the oracle's sequential solve; (c) the
result of a one-process Solve() of the same model; (d) the counters eval_round implies, so that a case cannot silently
stop sharding:
  - a sharded round issues one all-gather, the root round none, and the node-slot path adds one all-reduce per poll:
    collectives == rounds - 1 on the resident and single-tableau paths, >= rounds - 1 with slots;
  - a rank counts the node LPs of its share of every sharded round plus those every rank runs (the root and, when more
    than the root was committed, the final re-solve f): sum over ranks of nodes_evaluated == one-process count +
    (n_ranks - 1) * (1 + f), and rank r's count never exceeds rank r - 1's; at width 1 the ranks >= 1 count 1 + f;
  - shard_policy = 0 on nodes that fit shared memory shards nothing: collectives == 0 and every rank counts the
    one-process nodes_evaluated; so do the roots that end the run and the enhanced / incremental services.
Timeout cases check (a), that the log is a prefix of the oracle's full log, and that 0.001 ms fires."""
import gzip
import hashlib
import json
import os
import signal
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from helpers import strip_timeouts

pytestmark = pytest.mark.gpu

WORKER = os.path.join(ROOT, "tests", "dist_edges_worker.py")
WORK_COUNTERS = {"nodes_evaluated", "nodes_pruned", "gpu_ms", "kernel_launches", "host_eval_ms", "host_commit_ms",
                 "host_root_ms", "host_final_ms", "node_kernel_ms", "slot_pivots", "slot_ms", "slot_bytes",
                 "cycle_redos_kernel", "cycle_redos_slots", "cycle_redos_pruned"}
OPT_NODE_SLOTS, OPT_NODE_LOG_CAP = 10, 14


def bundle_model(name: str) -> dict:
    with gzip.open(os.path.join(ROOT, "tests", "golden", "sanity_fixtures.json.gz"), "rb") as f:
        b = json.loads(f.read().decode())
    return strip_timeouts([x for x in b["fixtures"] if x["file"] == name][0]["model"])


def tiny_models() -> dict:
    """Roots that end the run at once (presolve off, so branch and cut sees them)."""
    off = {"presolve": False}
    return {
        "root_integral": {"optimize": "v", "opType": "max", "constraints": {"c": {"max": 3}},
                          "variables": {"x": {"v": 1, "c": 1}}, "ints": {"x": 1}, "options": off},
        "root_infeasible": {"optimize": "v", "opType": "max", "constraints": {"lo": {"min": 5}, "hi": {"max": 3}},
                            "variables": {"x": {"v": 1, "lo": 1, "hi": 1}}, "ints": {"x": 1}, "options": off},
        "root_unbounded": {"optimize": "v", "opType": "max", "constraints": {"c": {"max": 1}},
                           "variables": {"x": {"v": 1, "c": 1}, "y": {"v": 1, "c": -1}}, "ints": {"x": 1},
                           "options": off},
    }


def cases_for(world: int) -> list:
    from jslpsolver_b200 import problems
    cases = []

    def add(cid, model, kind, **kw):
        cases.append(dict(id=f"w{world}_{cid}", model=model, check=kind, **kw))

    deal_models = {"knapsack1": bundle_model("Knapsack 1.json"), "woodshop": bundle_model("Integer Wood Shop Problem.json"),
                   "stockcut": bundle_model("StockCuttingProblem.json"),
                   "random2": problems.random_mip_model(10, 7, seed=2)}
    for name, jm in deal_models.items():
        for width in (1, 2, 3, 5, 7, 16):
            add(f"deal_{name}_k{width}", jm, "resident1", width=width, shard_policy=1)
    add("policy0_knapsack1", deal_models["knapsack1"], "policy0", width=8, shard_policy=0)
    for k in (1, 2, 7):
        add(f"priority{k}", problems.priority_tie_mip_model(k), "priority", width=5, n_opt=k)
    add("priority8", problems.priority_tie_mip_model(8), "refusal", width=5, n_opt=8)
    add("single_knapsack1", deal_models["knapsack1"], "single", engine=2, width=7, shard_policy=0,
        options={OPT_NODE_SLOTS: 0})
    add("slots_engine2_knapsack1", deal_models["knapsack1"], "slots", engine=2, width=8, shard_policy=0)
    add("logcap2_knapsack1", deal_models["knapsack1"], "resident1", width=6, shard_policy=1,
        options={OPT_NODE_LOG_CAP: 2})
    add("max_nodes_knapsack1", deal_models["knapsack1"], "resident1", width=5, shard_policy=1, max_nodes=23)
    add("tolerance_knapsack", problems.knapsack_mip_model(30, 4, seed=7, tolerance=0.05), "resident1", width=7,
        shard_policy=1)
    keep = dict(deal_models["knapsack1"], options={"keep_solutions": True})
    add("keep_solutions_knapsack1", keep, "resident1", width=3, shard_policy=1)
    for name, jm in tiny_models().items():
        add(name, jm, "root", width=4, shard_policy=1)
    farm = bundle_model("LargeFarmMIP.json")
    add("timeout_tiny", dict(farm, timeout=0.001), "timeout", width=4, shard_policy=1, fires=True)
    add("timeout_moderate", dict(farm, timeout=20), "timeout", width=4, shard_policy=1, fires=False)
    for name, opts in (("enhanced", {"nodeSelection": "best-first", "branching": "most-fractional"}),
                       ("incremental", {"useIncremental": True})):
        add(f"service_{name}", dict(deal_models["woodshop"], options=opts), "service", width=4, shard_policy=1)
    if world == 3:
        add("slots_half_tie300", problems.half_tie_mip_model(300, seed=300), "slots", width=16, max_nodes=40)
        z = np.load(os.path.join(ROOT, "tests", "golden", "config5_knapsack.npz"))
        add("config5_knapsack", problems.knapsack_mip_model(1024, 512, seed=12345), "golden", width=8,
            max_nodes=int(z["max_nodes"]))
    return cases


def launch(world: int, cases: list, tmp, backend: str = "gloo", timeout: float = 900) -> dict:
    """Runs every case at `world` ranks in one torchrun launch; {case id: [(arrays, meta) of rank 0, 1, ...]}."""
    path = os.path.join(tmp, "cases.json")
    with open(path, "w") as f:
        json.dump([{k: v for k, v in c.items() if k != "check"} for c in cases], f)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nnodes=1", "--nproc-per-node", str(world),
           WORKER, path, str(tmp), "--backend", backend]
    p = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True)
    try:
        out, _ = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)  # torchrun and every rank it started
        out, _ = p.communicate()
        pytest.fail(f"world {world}: no result after {timeout} s\n{out[-4000:]}")
    assert p.returncode == 0, out[-6000:]
    res = {}
    for c in cases:
        ranks = []
        for r in range(world):
            z = np.load(os.path.join(tmp, f"{c['id']}.rank{r}.npz"))
            ranks.append(({k: z[k] for k in z.files if k != "meta"}, json.loads(str(z["meta"]))))
        res[c["id"]] = ranks
    return res


def local_solve(case: dict):
    """The one-process Solve() of the case: (result dict, lastBnbStatus, model.solutions)."""
    import jslpsolver_b200 as J
    s = J.Solver()
    s.engine = case.get("engine", 0)
    s.max_spec_batch = case.get("width", 0)
    s.options = dict(case.get("options") or {})
    inst = s._instance(case["model"], None)
    inst.max_nodes = case.get("max_nodes", 0)
    gsol = s._finish(inst, inst.solve(), True)
    return s._simplified(gsol), gsol._tableau.lastBnbStatus, s.lastSolvedModel.solutions


def bits(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


def assert_log_parity(gnl, onl, what):
    """Every field of every node bit for bit, the evaluation an infeasible node logs included."""
    assert gnl.shape == onl.shape, (what, gnl.shape, onl.shape)
    assert np.array_equal(bits(gnl), bits(onl)), what


def assert_identical_ranks(ranks, what):
    a0, m0 = ranks[0]
    assert m0.get("error") is None or all(m.get("error") == m0["error"] for _, m in ranks), (what, m0.get("error"))
    for r, (a, m) in enumerate(ranks[1:], 1):
        assert set(a) == set(a0), (what, r)
        for k in a0:
            assert a[k].shape == a0[k].shape and np.array_equal(bits(a[k]), bits(a0[k])), (what, r, k)
        for k in ("iterations", "evaluation", "result", "solutions", "nOpt", "error"):
            assert m.get(k) == m0.get(k), (what, r, k, m.get(k), m0.get(k))
        st, st0 = m.get("status") or {}, m0.get("status") or {}
        for k in st0:
            if k not in WORK_COUNTERS:
                assert bits(st[k]) == bits(st0[k]), (what, r, k, st[k], st0[k])


def assert_oracle_parity(case, a, m, what):
    from oracle import ref_model
    osol = ref_model.solve_full(case["model"], fast_cycles=True, node_log=1 << 20, max_nodes=case.get("max_nodes", 0))
    assert osol.tableau is not None, what
    assert_log_parity(a["node_log"], osol.tableau.node_log(), what)
    assert m["iterations"] == osol.state.bncIterations, what
    assert np.array_equal(bits(a["matrix"]), bits(osol.tableau.matrix())), what
    assert np.array_equal(a["vrow"], osol.tableau.maps()[0]) and np.array_equal(a["vcol"], osol.tableau.maps()[1]), what
    assert m["evaluation"] == float(osol.evaluation).hex(), (what, m["evaluation"], osol.evaluation)
    assert m["result"] == ref_model.simplify(osol), what
    return osol


def assert_counters(case, ranks, want_status, what):
    """The counter identities of the module docstring."""
    n = len(ranks)
    st = [m["status"] for _, m in ranks]
    nodes = [s["nodes_evaluated"] for s in st]
    f = 1 if st[0]["iterations"] > 1 else 0
    kind = case["check"]
    if kind in ("policy0", "root", "service"):
        assert all(s["collectives"] == 0 for s in st), (what, [s["collectives"] for s in st])
        assert nodes == [want_status.nodes_evaluated] * n, (what, nodes, want_status.nodes_evaluated)
        return
    assert sum(nodes) == want_status.nodes_evaluated + (n - 1) * (1 + f), (what, nodes, want_status.nodes_evaluated, f)
    assert nodes == sorted(nodes, reverse=True), (what, nodes)
    if case.get("width") == 1:
        assert nodes[1:] == [1 + f] * (n - 1), (what, nodes)
    if kind in ("slots", "golden"):  # every rank with a node of a sharded round ran it in a slot (rounds of 2 leave rank 2 idle)
        assert st[0]["collectives"] >= st[0]["rounds"] - 1, (what, st[0])
        assert st[0]["slot_pivots"] > 0, what
        assert all(s["slot_pivots"] > 0 for s in st if s["nodes_evaluated"] > 1 + f), (what, st)
    else:
        assert st[0]["collectives"] == st[0]["rounds"] - 1, (what, st[0]["collectives"], st[0]["rounds"])
    if kind in ("single", "priority"):
        assert all(s["slot_pivots"] == 0 and s["node_kernel_ms"] == 0 for s in st), what


def check_case(case, ranks):
    what = case["id"]
    assert_identical_ranks(ranks, what)
    a, m = ranks[0]
    kind = case["check"]
    if kind == "refusal":  # nOpt > 7: refused on every rank, before any collective
        assert m["nOpt"] == case["n_opt"] and "more than 7 optional objectives" in (m["error"] or ""), (what, m)
        return
    assert m["error"] is None, (what, m["error"])
    if kind == "timeout":
        from oracle import ref_model
        full = ref_model.solve_full(strip_timeouts(case["model"]), fast_cycles=True, node_log=1 << 20)
        onl, gnl = full.tableau.node_log(), a["node_log"]
        assert len(gnl) == m["iterations"] <= len(onl), what
        assert_log_parity(gnl, onl[:len(gnl)], what)
        assert m["status"]["timed_out"] == (1 if len(gnl) < len(onl) else m["status"]["timed_out"]), what
        if case["fires"]:
            assert m["status"]["timed_out"] == 1, what
        return
    if kind == "golden":
        z = np.load(os.path.join(ROOT, "tests", "golden", "config5_knapsack.npz"))
        assert_log_parity(a["node_log"], z["node_log"], what)
        assert hashlib.sha256(np.ascontiguousarray(a["matrix"]).tobytes()).hexdigest() == str(z["final_matrix_sha"])
    else:
        osol = assert_oracle_parity(case, a, m, what)
    res, want_status, sols = local_solve(case)
    assert m["result"] == res, (what, m["result"], res)
    assert m["solutions"] == sols, what
    if kind == "priority":
        assert m["nOpt"] == case["n_opt"], what
        onl = osol.tableau.node_log()
        inc = onl[onl[:, 4] == 1]
        assert (inc[:, 3] == inc[-1, 3]).sum() >= 2, (what, inc)  # a later tie replaced the first incumbent
    if kind == "root":
        assert m["iterations"] == 1, what
    assert_counters(case, ranks, want_status, what)


@pytest.fixture(scope="module", params=[2, 3, 4], ids=lambda w: f"world{w}")
def sharded(request, tmp_path_factory):
    world = request.param
    cases = cases_for(world)
    return cases, launch(world, cases, tmp_path_factory.mktemp(f"dist{world}"))


def test_every_case_on_one_gpu(sharded):
    cases, res = sharded
    failures = []
    for case in cases:
        try:
            check_case(case, res[case["id"]])
        except AssertionError as e:
            failures.append(f"{case['id']}: {e}")
        st = [m.get("status") or {} for _, m in res[case["id"]]]
        print(case["id"], "rounds", st[0].get("rounds"), "collectives", st[0].get("collectives"),
              "nodes", [s.get("nodes_evaluated") for s in st], "pruned", [s.get("nodes_pruned") for s in st],
              "slot_pivots", [s.get("slot_pivots") for s in st])
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("world", [2, 3, 4])
def test_nccl_deals_slots_and_collectives(world, tmp_path):
    """The deal and slot cases over the in-library NCCL communicator, one GPU per rank, and the communicator's own
    collectives at 1 byte, 127 bytes, past its first 64 KiB buffer, and n = 0."""
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs (NCCL cannot put two ranks on one device)")
    cases = [c for c in cases_for(world)
             if c["check"] in ("slots", "golden") or c["id"].split("_", 1)[1].startswith("deal_")]
    cases.append({"id": f"w{world}_comm", "kind": "comm", "check": "comm"})
    res = launch(world, cases, tmp_path, backend="nccl")
    failures = []
    for case in cases:
        try:
            if case["check"] == "comm":
                assert all(m["ok"] and m["error"] is None for _, m in res[case["id"]]), res[case["id"]]
            else:
                check_case(case, res[case["id"]])
        except AssertionError as e:
            failures.append(f"{case['id']}: {e}")
    assert not failures, "\n".join(failures)

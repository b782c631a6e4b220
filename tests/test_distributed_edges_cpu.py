"""The sharded branch and cut's round logic without a GPU: N simulated ranks (tests/cpp/shard_replay.cpp) run the
product's speculation, deal, wire record and commit rule (jslp_frontier.h) over node results from the C oracle, and
every rank must commit the oracle's sequential node log bit for bit, at every world size from 1 to 8 and every
speculation width from 1 to 17, with and without optional objectives on the wire.  Also the wire record's round trip
at its edge values, the deal helpers, and the gloo all-gather hook at worlds 3 and 4."""
import json
import os
import socket
import subprocess

import numpy as np
import pytest

from conftest import ROOT, load_bundle
from helpers import strip_timeouts
from jslpsolver_b200 import problems


@pytest.fixture(scope="module")
def shard_exe(tmp_path_factory):
    exe = tmp_path_factory.mktemp("shard") / "shard_replay"
    p = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "include"),
                        "-I", os.path.join(ROOT, "jslpsolver_b200", "csrc"), "-o", str(exe),
                        os.path.join(ROOT, "tests", "cpp", "shard_replay.cpp")], capture_output=True, text=True)
    assert p.returncode == 0 and not p.stderr.strip(), p.stderr  # builds without a warning
    return exe


def test_wire_record_and_deal_helpers(shard_exe):
    """Every NodeEval field crosses to_wire / from_wire bit for bit (signed zeros, infinities, subnormals, NaN payloads,
    branch_var -1 and INT_MAX, pivots 2^31 - 1), opt0[7] has no slot on the wire, and for 1..8 ranks and rounds of 0..40
    nodes the deal gives every node its own record inside its own rank's block."""
    p = subprocess.run([str(shard_exe), "selftest"], capture_output=True, text=True)
    assert p.returncode == 0 and "SHARD SELFTEST OK" in p.stdout, p.stdout + p.stderr


def oracle_tableau(jm: dict, node_log: int = 0, max_nodes: int = 0):
    """The oracle's root tableau of jm as branch and cut sees it (presolve off), with its optional objectives."""
    from oracle import ref_model as R
    model = R.RefModel().loadJson(jm)
    M, vrow, vcol, prios, rc = model.build_tableau()
    unres = np.zeros(M.shape[0] + M.shape[1] - 2, dtype=np.uint8)
    for i in model.unrestrictedVariables:
        unres[i] = 1
    tab = R.OracleTableau(M, vrow, vcol, precision=model.precision, unrestricted=unres,
                          integers=[v.index for v in model.integerVariables], opt_rc=rc,
                          check_cycles=model.checkForCycles, is_min=model.isMinimization,
                          tolerance=model.tolerance or 0.0, max_nodes=max_nodes, node_log=node_log)
    return model, tab


def replay_shards(exe, jm: dict, n_ranks: int, width: int, max_nodes: int = 0):
    """Every simulated rank's (node log, iterations, best cut count, node LPs it evaluated) over jm."""
    model, tab = oracle_tableau(jm)
    p = subprocess.Popen([str(exe)], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
    p.stdin.write(f"{float(model.tolerance or 0)!r} {int(model.isMinimization)} {max_nodes} {width} {n_ranks} "
                  f"{tab.nOpt}\n")
    p.stdin.flush()
    ranks = []
    while True:
        line = p.stdout.readline().split()
        assert line, f"shard_replay exited with {p.wait()}"
        if line[0] == "EVAL":
            v = line[2:]
            cuts = [(int(v[3 * i]), int(v[3 * i + 1]), float(v[3 * i + 2])) for i in range(int(line[1]))]
            before = tab.state().totalPivots
            st = tab.apply_cuts(cuts)
            integral = int(st.feasible and tab.is_integral())
            var, val = tab.most_fractional() if st.feasible and not integral else (-1, 0.0)
            optimal = int(st.feasible and st.bounded)
            # the product reads optionalObjectives[o].reducedCosts[0] of feasible nodes only
            opt = tab.optional()[:, 0] if st.feasible else np.zeros(tab.nOpt)
            p.stdin.write(f"{st.feasible} {st.bounded} {optimal} {integral} {var} {val!r} {st.evaluation!r} "
                          f"{st.totalPivots - before}" + "".join(f" {float(x)!r}" for x in opt) + "\n")
            p.stdin.flush()
        elif line[0] == "SAVE":
            tab.save()
            p.stdin.write("ok\n")
            p.stdin.flush()
        elif line[0] == "RANK":
            log = np.array([[float(x) for x in p.stdout.readline().split()] for _ in range(int(line[3]))])
            it, nbest, evals = (int(x) for x in p.stdout.readline().split()[1:])
            ranks.append((log.reshape(-1, 8), it, nbest, evals))
            if len(ranks) == n_ranks:
                assert p.wait() == 0
                return ranks


def oracle_run(jm: dict, max_nodes: int = 0):
    """The oracle's sequential branch and cut over the same tableau: (node log, iterations, best cut count)."""
    _, tab = oracle_tableau(jm, node_log=1 << 16, max_nodes=max_nodes)
    st = tab.branch_and_cut()
    return tab.node_log(), st.bncIterations, len(tab.best_cuts()) if st.isIntegral else None


def bundle_mips(limit_vars: int = 40):
    b = load_bundle()
    return [strip_timeouts(f["model"]) for f in b["fixtures"]
            if (f["model"].get("ints") or f["model"].get("binaries")) and len(f["model"]["variables"]) <= limit_vars]


CASES = ([(jm.get("name") or f"bundle{i}", jm, 0) for i, jm in enumerate(bundle_mips())] +
         [(f"random_mip_{s}", problems.random_mip_model(10, 7, seed=s), 0) for s in (2, 29, 36, 64)] +
         [("half_tie_24_cap60", problems.half_tie_mip_model(24, group=4, seed=5), 60)] +
         [(f"priority_tie_{k}", problems.priority_tie_mip_model(k), 0) for k in (1, 2, 7)])


@pytest.mark.parametrize("name,jm,max_nodes", CASES, ids=[c[0] for c in CASES])
def test_every_rank_commits_the_oracle_log(shard_exe, name, jm, max_nodes):
    """At 1..8 ranks and widths 1..17 (rounds smaller than the world, ragged last blocks, empty ranks) every rank's node
    log is the oracle's bit for bit.  The ranks take the rounds one rank takes and split them: their node LPs add up to
    the one-rank count (the root counted once, on rank 0; every rank solves it in the product), and within a round
    rank r gets ceil((n - r) / n_ranks) of its n nodes, so the later ranks never get more."""
    want, it, nbest = oracle_run(jm, max_nodes)
    assert len(want) > 1, name  # the root branches: later rounds are sharded
    for width in range(1, 18):
        total = None
        for n_ranks in range(1, 9):
            ranks = replay_shards(shard_exe, jm, n_ranks, width, max_nodes)
            for r, (log, rit, rbest, _) in enumerate(ranks):
                what = (name, n_ranks, width, r)
                assert rit == it, what
                assert log.shape == want.shape and np.array_equal(log.view(np.uint64), want.view(np.uint64)), what
                assert nbest is None or rbest == nbest, what
            evals = [e for *_, e in ranks]
            total = sum(evals) if total is None else total
            assert sum(evals) == total, (name, width, evals)
            shares = [evals[0] - 1] + evals[1:]
            assert shares == sorted(shares, reverse=True), (name, width, evals)
            if width == 1:  # rounds of one node: rank 0 evaluates every node, the others none
                assert evals[1:] == [0] * (n_ranks - 1), (name, n_ranks, evals)


@pytest.mark.parametrize("k", [1, 2, 7, 8])
def test_priority_model_has_one_optional_objective_per_priority(k):
    """priority_tie_mip_model(k) has exactly k optional objectives; a second soft constraint at a priority already in
    use adds none.  The oracle's incumbent is decided by them: its node log has a later incumbent at the same
    evaluation as an earlier one, which only the optional-objective comparison lets through."""
    from oracle import ref_model as R
    jm = problems.priority_tie_mip_model(k)
    assert len(R.RefModel().loadJson(jm).build_tableau()[3]) == k
    twin = json.loads(json.dumps(jm))
    twin["constraints"]["extra"] = {"max": 3.0, "priority": k, "weight": 2.0}
    twin["variables"]["x0"]["extra"] = 1.0
    assert len(R.RefModel().loadJson(twin).build_tableau()[3]) == k
    log, _, _ = oracle_run(jm)
    inc = log[log[:, 4] == 1]
    best = inc[-1, 3]
    assert (inc[:, 3] == best).sum() >= 2, inc


# ---- the gloo all-gather hook at three and four ranks ---------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _hook_worker(rank, world, port, sizes, out_dir):
    import sys
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    from jslpsolver_b200 import distributed as D
    cb, keep = D.make_all_gather_hook()
    ok = True
    for rnd, n in enumerate(sizes):  # successive rounds of different sizes through the same hook
        buf = np.full(world * n, 0xA5, dtype=np.uint8)  # other ranks' blocks hold stale bytes before the gather
        buf[rank * n:(rank + 1) * n] = (np.arange(n) * (rank + 3) + 7 * rnd) % 251
        ok = ok and cb(None, buf.ctypes.data, n) == 0
        for r in range(world):
            ok = ok and np.array_equal(buf[r * n:(r + 1) * n], ((np.arange(n) * (r + 3) + 7 * rnd) % 251).astype(np.uint8))
    with open(os.path.join(out_dir, f"rank{rank}.json"), "w") as f:
        json.dump({"ok": bool(ok)}, f)
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [3, 4])
def test_all_gather_hook_world3_and_4_gloo(tmp_path, world):
    import torch.multiprocessing as mp
    sizes = [1, 127, 128 * 3, 200 * 1024 + 3, 1, 129]
    mp.spawn(_hook_worker, args=(world, _free_port(), sizes, str(tmp_path)), nprocs=world, join=True)
    for r in range(world):
        assert json.load(open(tmp_path / f"rank{r}.json"))["ok"]

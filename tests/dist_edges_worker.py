#!/usr/bin/env python
"""One rank of the sharded branch-and-cut edge cases (tests/test_gpu_dist_edges.py launches it; not a test module):

  python -m torch.distributed.run --standalone --nproc-per-node N tests/dist_edges_worker.py CASES.json OUT_DIR
      [--backend gloo|nccl]

Solves every case of CASES.json with the tableau's rounds sharded over the ranks (Tableau.distributed) and writes
OUT_DIR/<case>.rank<r>.npz: the node log, every lastBnbStatus field, the iterations and best cuts, the final tableau
and its labels, the Solve() result and model.solutions.  gloo (the default) puts every rank on cuda:0 with the
all-gather hook; nccl gives each rank its own device and the in-library communicator.  A case of kind "comm" checks
jslp_comm_all_gather / jslp_comm_all_reduce_min directly (nccl only).  Every collective times out after 120 s, so a
rank that diverges fails with an error instead of waiting forever."""
import json
import os
import sys
import traceback
from datetime import timedelta

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def status_dict(b) -> dict:
    return {name: getattr(b, name) for name, _ in b._fields_}


def solve_case(J, case: dict):
    """(arrays, meta) of one sharded solve."""
    import numpy as np
    s = J.Solver()
    s.engine = case.get("engine", 0)
    s.max_spec_batch = case.get("width", 0)
    s.node_slots = case.get("node_slots")
    s.slot_steps = case.get("slot_steps")
    s.options = {int(k): v for k, v in (case.get("options") or {}).items()}
    inst = s._instance(case["model"], None)
    inst.max_nodes = case.get("max_nodes", 0)
    inst.tableau.distributed = True
    inst.tableau.shard_policy = case.get("shard_policy", 0)
    try:
        gsol = s._finish(inst, inst.solve(), True)
    except J.JslpError as e:  # refusals are results too: every rank must refuse alike
        return {}, {"error": str(e), "nOpt": int(getattr(inst.tableau, "nOpt", -1))}
    gt = gsol._tableau
    m = s.lastSolvedModel
    arrays = {"node_log": gt.node_log(), "matrix": np.ascontiguousarray(gt.matrix2d()),
              "vrow": np.asarray(gt.varIndexByRow), "vcol": np.asarray(gt.varIndexByCol),
              "best_cuts": np.array([(a, b, float(c)) for a, b, c in gt.bestCuts], dtype=np.float64).reshape(-1, 3)}
    meta = {"status": status_dict(gt.lastBnbStatus), "iterations": gt.branchAndCutIterations,
            "evaluation": gsol.evaluation.hex() if isinstance(gsol.evaluation, float) else gsol.evaluation,
            "result": s._simplified(gsol), "solutions": m.solutions, "nOpt": int(gt.nOpt), "error": None}
    return arrays, meta


def comm_case(J, rank: int, world: int):
    """jslp_comm_all_gather at 1 byte, 127 bytes and past comm_reserve's first 64 KiB, jslp_comm_all_reduce_min, and
    n = 0 (no collective: the buffer is left as it was)."""
    import numpy as np
    from jslpsolver_b200 import _lib, distributed as D
    from jslpsolver_b200.tableau import default_context
    ctx = default_context()
    comm = D.nccl_communicator(ctx)
    L = ctx.lib
    ok = True
    for n in (1, 127, 3 * 65536 + 5, 129):
        buf = np.full(world * n, 0x5A, dtype=np.uint8)
        buf[rank * n:(rank + 1) * n] = (np.arange(n) * (rank + 5) + n) % 253
        _lib.check(L.jslp_comm_all_gather(comm, buf.ctypes.data, n))
        for r in range(world):
            ok = ok and np.array_equal(buf[r * n:(r + 1) * n], ((np.arange(n) * (r + 5) + n) % 253).astype(np.uint8))
    for n in (1, 2, 9000):
        v = np.array([(k * 7 + rank * 3) % 11 - 5.5 for k in range(n)], dtype=np.float64)
        _lib.check(L.jslp_comm_all_reduce_min(comm, v.ctypes.data, n))
        want = np.min([[(k * 7 + r * 3) % 11 - 5.5 for k in range(n)] for r in range(world)], axis=0)
        ok = ok and np.array_equal(v, want)
    buf = np.arange(8, dtype=np.uint8)
    v = np.array([float(rank)])
    _lib.check(L.jslp_comm_all_gather(comm, buf.ctypes.data, 0))
    _lib.check(L.jslp_comm_all_reduce_min(comm, v.ctypes.data, 0))
    ok = ok and np.array_equal(buf, np.arange(8, dtype=np.uint8)) and v[0] == rank
    return {}, {"ok": bool(ok), "error": None}


def main():
    import numpy as np
    import torch
    import torch.distributed as dist
    cases_path, out_dir = sys.argv[1], sys.argv[2]
    backend = sys.argv[sys.argv.index("--backend") + 1] if "--backend" in sys.argv else "gloo"
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if backend == "gloo":  # every rank on cuda:0, the all-gather hook over gloo
        local = 0
        os.environ["JSLP_DEVICE"] = "0"
    else:
        os.environ["JSLP_DEVICE"] = str(local)
    torch.cuda.set_device(local)
    if backend == "nccl":
        dist.init_process_group("nccl", device_id=torch.device("cuda", local), timeout=timedelta(seconds=120))
    else:
        dist.init_process_group("gloo", timeout=timedelta(seconds=120))
    import jslpsolver_b200 as J
    with open(cases_path) as f:
        cases = json.load(f)
    for case in cases:
        try:
            arrays, meta = comm_case(J, rank, world) if case.get("kind") == "comm" else solve_case(J, case)
        except Exception:  # the other ranks may now wait in a collective: end this rank so the launch fails fast
            meta = {"error": traceback.format_exc(), "rank": rank, "world": world, "backend": backend}
            np.savez(os.path.join(out_dir, f"{case['id']}.rank{rank}.npz"), meta=np.array(json.dumps(meta)))
            raise
        meta.update(rank=rank, world=world, backend=backend)
        np.savez(os.path.join(out_dir, f"{case['id']}.rank{rank}.npz"), meta=np.array(json.dumps(meta)), **arrays)
    from jslpsolver_b200 import distributed as D
    D.destroy_communicators()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

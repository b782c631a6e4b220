"""Time near-optimal variability on one GPU: the bound tableau (jslp_bound_create), the batch of target LPs on it and
the whole Solution.variability(gap=...) call, against the way a user gets the same numbers without it.

For each size, builds the seeded LP with planted alternative optima (problems.alternative_optima_model) as a JSON model
and solves it once with Solve(model, full=True).  Then, each timed on the host clock around work that ends in a
synchronise:
  bound   GpuTableau.bound(t) of the solved tableau (--reps times after one warm-up)
  batch   one scenario_batch of every target of DESIGN.md section 2i rule 3 on the bound tableau (once): LPs, pivots
          per target, statuses, kernel launches and the path the batch took (shared memory: about one launch per
          chunk of targets; single tableau: a restore, an edit and a simplex per target)
  call    the whole Solution.variability(gap=...) (--call-reps times)
  user    the alternative a user has without it: the objective bound `objective >= z - t` added to the JSON model as
          a constraint and one cold Solve() per target, for a sample of --user-samples structural variables, max and
          min in turn (each answer listed beside the call's range end; a cold solve can also end "infeasible", since
          it starts from the all-slack basis with the bound row violated)
Prints one JSON line per size with the device name and power limit read in the same run.

    python scripts/near_optimal_bench.py [--sizes 150x120,550x600,2000x2000] [--gap 0.01] [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_conditions():
    try:
        out = subprocess.run(["nvidia-smi", "-i", os.environ.get("JSLP_DEVICE", "0"),
                              "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout
        pw, mx, cur = (float(x) for x in out.strip().splitlines()[0].split(","))
        return {"power_limit_w": pw, "clocks_max_sm_mhz": mx, "clocks_sm_mhz": cur}
    except Exception:
        return {"power_limit_w": None, "clocks_max_sm_mhz": None, "clocks_sm_mhz": None}


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def run_size(n_vars, n_cons, gap, reps, call_reps, samples, seed):
    import numpy as np
    import jslpsolver_b200 as J
    from jslpsolver_b200 import problems
    jm = problems.alternative_optima_model(n_vars, n_cons, seed)
    solve_ms, sol = timed(lambda: J.Solve(jm, full=True))
    assert sol.feasible and sol.bounded, "the benchmark LP has no optimum"
    g, m = sol._tableau, sol._tableau.model
    rhs, cost, vrow, vcol = g.final_state()
    t = max(0.0, gap * abs(float(cost[0])))
    H, W = g.height, g.width

    g.bound(t).close()  # warm-up: allocator, kernel load
    bound_ms = []
    for _ in range(reps):
        ms, b = timed(lambda: g.bound(t))
        bound_ms.append(ms)
        b.close()

    basic = {int(x) for x in vrow[1:]}
    labels = [v.index for v in m.variables] + [c.index for c in m.constraints]
    targets = [(lab, s) for lab in labels for s in ((-1, 1) if lab in basic else (1,))]
    b = g.bound(t)
    launches0 = g.context.launches
    batch_ms, out = timed(lambda: b.scenario_batch([(1, lab, float(-s)) for lab, s in targets],
                                                   list(range(len(targets) + 1)), check_cycles=True))
    launches = g.context.launches - launches0
    b.close()
    pivots = out["p1"] + out["p2"]

    call_ms = []
    for _ in range(call_reps):
        ms, v = timed(lambda: sol.variability(gap=gap))
        call_ms.append(ms)
    assert v["lps"] == len(targets) and v["allowance"] == t

    # the user's alternative: the bound as a JSON constraint, one cold Solve() per sampled target
    z = -float(cost[0])  # result = -sigma * M[0,0], the model maximises
    bounded = dict(jm, constraints=dict(jm["constraints"], objective_bound={"min": z - t}))
    bounded["variables"] = {k: dict(a, objective_bound=a.get(jm["optimize"], 0)) for k, a in jm["variables"].items()}
    ids = [x.id for x in m.variables]
    picks = [ids[int(k)] for k in np.linspace(0, len(ids) - 1, samples)] if samples else []
    user_ms, user = [], []
    for k, vid in enumerate(picks):
        sense = "max" if k % 2 == 0 else "min"
        model = dict(bounded, optimize="target", opType=sense)
        model["variables"] = {x: dict(a, target=1 if x == vid else 0) for x, a in bounded["variables"].items()}
        ms, res = timed(lambda: J.Solve(model))
        user_ms.append(ms)
        want = v["variables"][vid][sense]
        got = float(res["result"]) if res.get("feasible") and res.get("bounded") else None
        user.append({"id": vid, "sense": sense, "range_end": want, "cold_solve": got,
                     "feasible": bool(res.get("feasible")), "ms": ms,
                     "agrees": got is not None and abs(got - want) <= 1e-6 * max(1.0, abs(want))})

    return {"tableau": f"{H}x{W}", "bound_tableau": f"{H + 1}x{W}", "gap": gap, "allowance": t, "solve_ms": solve_ms,
            "bound_ms": spread(bound_ms), "lps": len(targets), "batch_ms": batch_ms, "launches": launches,
            "path": "shared-memory" if launches < len(targets) else "single-tableau",
            "pivots_per_target": {"mean": float(pivots.mean()), "max": int(pivots.max()), "total": int(pivots.sum())},
            "statuses": {str(s): int((out["status"] == s).sum()) for s in range(4)},
            "call_ms": spread(call_ms), "unique": v["unique"], "exact": v["exact"],
            "user_solve_ms": spread(user_ms) if user_ms else None, "user_samples": len(picks),
            "user_est_total_ms": statistics.median(user_ms) * len(targets) if user_ms else None,
            "user_targets": user, "reps": reps, "call_reps": call_reps}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="150x120,550x600,2000x2000", help="comma-separated VARSxCONS")
    ap.add_argument("--gap", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--call-reps", type=int, default=2)
    ap.add_argument("--user-samples", type=int, default=4)
    ap.add_argument("--seed", type=int, default=12345)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only measures on the GPU")
    dev, cond = torch.cuda.get_device_name(0), gpu_conditions()
    for shape in a.sizes.split(","):
        nv, nc = (int(x) for x in shape.split("x"))
        out = run_size(nv, nc, a.gap, a.reps, a.call_reps, a.user_samples, a.seed)
        out.update(device=dev, **cond)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

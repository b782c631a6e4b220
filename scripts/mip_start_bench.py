"""Time MIP starts on one GPU: cold Solve() against Solve(model, start=...), alternated, on knapsack and random-MIP
models from problems.py that a cold solve finishes.

Each model is seeded three ways:
  own      the cold run's own plan: the upper bound of the gain
  capped   the plan of a run capped at --cap tree nodes: a realistic incumbent (skipped when that run found none)
  noisy    yesterday's plan: the optimal plan of the same model with every weight x (1 + 0.02 N(0,1)), re-solved on
           today's weights (rolling re-solve); a start the host rejects or the dive cannot complete is reported as such
For each arm it reports tree nodes (branchAndCutIterations), start nodes, pruned nodes, kernel launches and wall time
(host clock around Solve(), which ends in a synchronise), and whether the results agree to 1e-9 relative.  Prints one
JSON line per case with the device name and power limit read in the same call.

    python scripts/mip_start_bench.py [--models knapsack:24x8,knapsack:32x12,random:40x20] [--reps 3] [--cap 300]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", os.environ.get("JSLP_DEVICE", "0"), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def model_of(spec: str, seed: int) -> dict:
    from jslpsolver_b200 import problems
    kind, size = spec.split(":")
    a, b = (int(x) for x in size.split("x"))
    if kind == "knapsack":
        return problems.knapsack_mip_model(a, b, seed=seed)
    if kind == "random":
        return problems.random_mip_model(a, b, seed=seed)
    raise SystemExit(f"unknown model kind {kind!r}")


def noisy(jm: dict, seed: int) -> dict:
    """The same model with every constraint coefficient x (1 + 0.02 N(0,1))."""
    import numpy as np
    rng = np.random.default_rng(seed)
    out = copy.deepcopy(jm)
    for coefs in out["variables"].values():
        for k in coefs:
            if k != jm["optimize"] and k in jm["constraints"]:
                coefs[k] = float(coefs[k]) * (1 + 0.02 * rng.standard_normal())
    return out


def plan_of(res: dict, jm: dict) -> dict:
    return {k: v for k, v in res.items() if k in jm["variables"]}


def solve(jm: dict, start=None, max_nodes: int = 0):
    """(simplified result, ms, tree nodes, pruned, launches, mipStart or None) of one Solve() call."""
    import jslpsolver_b200 as J
    S = J.Solver()
    m = S._instance(copy.deepcopy(jm), None)
    m.max_nodes = max_nodes
    t0 = time.perf_counter()
    sol = m.solve(start=start) if start is not None else m.solve()
    ms = 1e3 * (time.perf_counter() - t0)
    S._finish(m, sol, True)
    st = m.tableau.lastBnbStatus
    return (S._simplified(sol), ms, int(st.iterations), int(st.nodes_pruned), int(st.kernel_launches),
            getattr(sol, "mipStart", None))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="knapsack:24x8,knapsack:32x12,knapsack:40x16,random:40x20,random:60x30")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cap", type=int, default=300)
    ap.add_argument("--seed", type=int, default=11)
    args = ap.parse_args()
    import torch
    dev = torch.cuda.get_device_name(0)
    watts = power_limit_w()
    for spec in args.models.split(","):
        jm = model_of(spec, args.seed)
        cold, *_ = solve(jm)
        yesterday = noisy(jm, args.seed + 1)
        capped, _, capped_nodes, *_ = solve(jm, max_nodes=args.cap)
        seeds = {"own": plan_of(cold, jm), "noisy": plan_of(solve(yesterday)[0], jm)}
        if capped.get("isIntegral") and capped_nodes >= args.cap:
            seeds["capped"] = plan_of(capped, jm)
        for arm, start in seeds.items():
            rows = {"cold": [], "seeded": []}
            for _ in range(args.reps):  # alternated: cold, seeded, cold, seeded, ...
                rows["cold"].append(solve(jm))
                rows["seeded"].append(solve(jm, start))
            c, s = rows["cold"][-1], rows["seeded"][-1]
            rep = s[5]
            agree = c[0]["feasible"] == s[0]["feasible"] and (
                not c[0]["feasible"] or abs(c[0]["result"] - s[0]["result"]) <= 1e-9 * max(1.0, abs(c[0]["result"])))
            print(json.dumps({
                "model": spec, "seed_kind": arm, "device": dev, "power_limit_w": watts,
                "cold": {"tree_nodes": c[2], "pruned": c[3], "launches": c[4],
                         "ms": sorted(r[1] for r in rows["cold"])[len(rows["cold"]) // 2]},
                "seeded": {"tree_nodes": s[2], "start_nodes": rep["nodes"], "pruned": s[3], "launches": s[4],
                           "ms": sorted(r[1] for r in rows["seeded"])[len(rows["seeded"]) // 2],
                           "start_status": rep["starts"][0]["status"], "improved": rep["improved"]},
                "results_agree": agree}), flush=True)


if __name__ == "__main__":
    main()

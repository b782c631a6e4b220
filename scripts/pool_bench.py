"""Pool() on the device against the sequential restatement (tests/pool_oracle.py, on the CPU) on the same inputs.
Workloads: LargeFarmMIP from the fixture bundle (at gap 0), the knapsack families of problems.py and a mid-size random
MIP (at gap 0.02, so that k plans exist within the allowance), each at k = 10 and k = 100 with at most --max-nodes
committed region LPs.  Per workload and k:

  ms/call      host clock around Pool() (it ends in a device synchronise), best of --runs after one warm-up call
  lps, nodes   region LPs evaluated / committed; lps / nodes is the speculation that was wasted
  LPs/s        lps over the call time;  launches and rounds (jslp_pool_batch calls) per call
  pivots/LP    mean phase-1 + phase-2 pivots of an evaluated region LP (every region starts from the initial tableau)
  cpu ms       one call of the sequential search on the C restatement

GPU name, power limit and clocks are read in the same run.  Usage: python scripts/pool_bench.py [--runs 3]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info() -> str:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def workloads():
    from conftest import load_bundle
    from jslpsolver_b200 import problems
    farm = [f["model"] for f in load_bundle()["fixtures"] if f["file"] == "LargeFarmMIP.json"][0]
    return [("LargeFarmMIP", farm, 0.0),
            ("knapsack 40", problems.single_knapsack_model(40, seed=3), 0.02),
            ("knapsack 40x5", problems.knapsack_mip_model(40, 5, seed=3), 0.02),
            ("random MIP 30x20", problems.random_mip_model(30, 20, seed=17, integer_fraction=0.5), 0.02)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--max-nodes", type=int, default=20000)
    ap.add_argument("--width", type=int, default=None)
    args = ap.parse_args()
    import jslpsolver_b200 as J
    import pool_oracle as O
    from oracle import ref_model
    from jslpsolver_b200.tableau import default_context
    ref_model.build_oracle()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name, jm, gap in workloads():
        for k in (10, 100):
            J.Pool(jm, k=k, gap=gap, max_nodes=args.max_nodes, width=args.width)  # warm-up
            best, r = None, None
            for _ in range(args.runs):
                default_context().sync()
                t0 = time.perf_counter()
                r = J.Pool(jm, k=k, gap=gap, max_nodes=args.max_nodes, width=args.width)
                dt = time.perf_counter() - t0
                best = dt if best is None else min(best, dt)
            t0 = time.perf_counter()
            o = O.pool(jm, k=k, gap=gap, max_nodes=args.max_nodes)
            cpu = time.perf_counter() - t0
            same = [s["values"] for s in r["solutions"]] == [s["values"] for s in o["solutions"]] and \
                r["nodes"] == o["nodes"] and r["stop"] == o["stop"]
            print(json.dumps({"workload": name, "k": k, "gap": gap, "found": len(r["solutions"]), "stop": r["stop"],
                              "ms_per_call": round(1e3 * best, 2), "lps": r["lps"], "nodes": r["nodes"],
                              "lps_per_node": round(r["lps"] / r["nodes"], 3), "lps_per_s": round(r["lps"] / best),
                              "launches": r["launches"], "rounds": r["rounds"],
                              "pivots_per_lp": round(r["pivots"] / r["lps"], 1), "cpu_ms": round(1e3 * cpu, 2),
                              "same_as_sequential": same}), flush=True)


if __name__ == "__main__":
    main()

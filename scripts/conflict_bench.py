"""Conflict() on the device against the sequential restatement (tests/conflict_oracle.py, on the CPU) on the same
inputs.  Workloads: planted parity conflicts of problems.py at a few sizes (the last beyond shared memory, so its node
LPs run on the single-tableau path) and Sudoku4x4 with a contradictory clue.  Per workload:

  ms/call      host clock around Conflict() (it ends in a device synchronise), best of --runs after one warm-up call
  tests        feasibility searches run;  nodes / lps: node LPs committed / evaluated
  wasted       lps - nodes: speculative node LPs of searches that ended before reaching them
  LPs/s        lps over the call time;  launches per call
  pivots/LP    mean phase-1 pivots of an evaluated node LP (every node starts from the initial tableau's rows)
  cpu ms       one call of the sequential restatement on the C oracle

GPU name, power limit and clocks are read in the same run.  Usage: python scripts/conflict_bench.py [--runs 3]"""
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
    from jslpsolver_b200 import problems
    from test_conflict_cpu import sudoku_with_contradictory_clue
    return [("planted 30x40 k=4", problems.planted_integer_conflict_model(30, 40, 4, 3)),
            ("planted 60x120 k=4", problems.planted_integer_conflict_model(60, 120, 4, 8)),
            ("planted 100x200 k=5", problems.planted_integer_conflict_model(100, 200, 5, 9)),
            ("planted 80x400 k=3 (beyond shared memory)", problems.planted_integer_conflict_model(80, 400, 3, 5)),
            ("Sudoku4x4 + clue", sudoku_with_contradictory_clue())]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    import jslpsolver_b200 as J
    import conflict_oracle as O
    from oracle import ref_model
    from jslpsolver_b200.tableau import default_context
    ref_model.build_oracle()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name, jm in workloads():
        J.Conflict(jm)  # warm-up
        best, r = None, None
        for _ in range(args.runs):
            default_context().sync()
            t0 = time.perf_counter()
            r = J.Conflict(jm)
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        t0 = time.perf_counter()
        o = O.conflict(jm)
        cpu = time.perf_counter() - t0
        same = {k: v for k, v in r.items() if k not in ("tests", "nodes", "lps", "launches", "pivots")} == O.named(o)
        print(json.dumps({"workload": name, "rows": len(r["constraints"]) + len(r["bounds"]),
                          "integers": len(r["integers"]), "ms_per_call": round(1e3 * best, 2), "tests": r["tests"],
                          "nodes": r["nodes"], "lps": r["lps"], "wasted": r["lps"] - r["nodes"],
                          "lps_per_s": round(r["lps"] / best), "launches": r["launches"],
                          "pivots_per_lp": round(r["pivots"] / r["lps"], 1), "cpu_ms": round(1e3 * cpu, 2),
                          "same_as_sequential": same}), flush=True)


if __name__ == "__main__":
    main()

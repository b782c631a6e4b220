"""LexicographicMIP() on the device against the sequential restatement (tests/lexicographic_mip_oracle.py, on the CPU)
and against what a user does without it: one Solve() per level (presolve off), each earlier objective written in as a
constraint row at its optimum minus / plus its allowance.  Workloads: a 40x5 multi-dimensional knapsack with two seeded
extra objectives at gap 0 and 0.01, and Sudoku4x4 (a feasibility model, so every plan is optimal at level 1) with one
seeded extra objective.  The three ways run alternated, once each per run, --runs times after one warm-up.  Per
workload and gap:

  ms           host clock around the call (each ends in a device synchronise or runs on the CPU), best of --runs
  launches     device launches of one LexicographicMIP() call;  lps, nodes, rounds, pivots its counters
  cpu ms       the restatement on the C oracle; "same" says its result equals the device's key for key
  solve ms     the one-Solve()-per-level chain; "agrees" says its optima equal the device's within 1e-6 relative

GPU name, power limit and clocks are read in the same run.  Usage: python scripts/lexicographic_mip_bench.py [--runs 5]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def workloads():
    from conftest import load_bundle
    from jslpsolver_b200 import problems
    from test_lexicographic_mip_cpu import with_extra
    sudoku = with_extra(next(f["model"] for f in load_bundle()["fixtures"] if f["file"] == "Sudoku4x4.json"), ["min"],
                        seed=2)
    return [("knapsack 40x5 + 2", with_extra(problems.knapsack_mip_model(40, 5, seed=3), ["min", "max"], seed=3),
             (0.0, 0.01)),
            ("Sudoku4x4 + 1", dict(sudoku, optimize={"feasible": "min", "extra1": "min"}), (0.0,))]


def by_solve(jm: dict, gap: float) -> list:
    """The level optima from one Solve() per level: objective k with every earlier objective j as a row at z_j -+ t_j
    (widened by 1e-9 relative, as the solver meets rows within its precision)."""
    import jslpsolver_b200 as J
    from jslpsolver_b200.model import object_keys
    keys = object_keys(jm["optimize"])
    rows, opts = dict(jm["constraints"]), []
    variables = {v: dict(spec) for v, spec in jm["variables"].items()}
    for k, key in enumerate(keys):
        sense = jm["optimize"][key]
        for spec in variables.values():
            spec["__level"] = spec.get(key, 0.0)
        r = J.Solve(dict(jm, constraints=rows, variables=variables, optimize="__level", opType=sense,
                         options={"presolve": False}))
        z = r["result"]
        opts.append(z)
        t = gap * abs(z)
        slack = 1e-9 * max(1.0, abs(z))
        rows[f"__obj{k}"] = {"min": z - t - slack} if sense == "max" else {"max": z + t + slack}
        for spec in variables.values():
            spec[f"__obj{k}"] = spec.get(key, 0.0)
    return opts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--width", type=int, default=None)
    args = ap.parse_args()
    import jslpsolver_b200 as J
    import lexicographic_mip_oracle as LMO
    from oracle import ref_model
    from pool_bench import gpu_info
    from jslpsolver_b200.tableau import default_context
    ref_model.build_oracle()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name, jm, gaps in workloads():
        for gap in gaps:
            r = J.LexicographicMIP(jm, gap=gap, width=args.width)  # warm-up
            by_solve(jm, gap)
            best = {"device": None, "cpu": None, "solve": None}
            for _ in range(args.runs):
                default_context().sync()
                t0 = time.perf_counter()
                r = J.LexicographicMIP(jm, gap=gap, width=args.width)
                t1 = time.perf_counter()
                # the restatement reproduces the device's counters at the device's width; a default width is one
                # wave of the level's tableau, which only the device knows, so the restatement runs at width 16 then
                o, _ = LMO.chain(jm, gap=gap, width=args.width or 16)
                t2 = time.perf_counter()
                naive = by_solve(jm, gap)
                default_context().sync()
                t3 = time.perf_counter()
                for k, dt in (("device", t1 - t0), ("cpu", t2 - t1), ("solve", t3 - t2)):
                    best[k] = dt if best[k] is None else min(best[k], dt)
            mine = [lv["optimum"] for lv in r["levels"]]
            same = all(r[k] == o[k] for k in ("feasible", "stop", "values", "objectives")) and \
                mine == [lv["optimum"] for lv in o["levels"]]
            agrees = len(naive) == len(mine) and all(abs(a - b) <= 1e-6 * max(1.0, abs(a), abs(b))
                                                     for a, b in zip(mine, naive))
            print(json.dumps({"workload": name, "gap": gap, "stop": r["stop"], "optima": mine,
                              "kinds": [lv["kind"] for lv in r["levels"]], "ms": round(1e3 * best["device"], 2),
                              "launches": r["launches"], "lps": r["lps"], "nodes": r["nodes"], "rounds": r["rounds"],
                              "pivots": r["pivots"], "cpu_ms": round(1e3 * best["cpu"], 2), "same": same,
                              "solve_ms": round(1e3 * best["solve"], 2), "agrees": agrees}), flush=True)


if __name__ == "__main__":
    main()

"""Variability() on the device against the sequential restatement (tests/mip_variability_oracle.py, on the CPU) and
against the naive way to the same ranges.  Workloads: Knapsack 1 from the fixture bundle, the knapsack families of
problems.py, a 30x20 random MIP, a 60x40 mixed MIP and Sudoku4x4, each at gap 0 and 0.01.  Per workload and gap:

  ms/call      host clock around Variability() (it ends in a device synchronise), best of --runs after one warm-up
  searches     target searches (two per reported variable and row)
  lps, nodes   node LPs evaluated / committed, the optimum search included
  LPs/s        lps over the call time;  launches and rounds (batch calls) per call
  pivots/LP    mean phase-1 + phase-2 pivots of an evaluated node LP (a target's nodes start from the bound tableau,
               warm; the optimum search's regions start from the initial tableau)
  cpu ms       one call of the restatement on the C oracle (models up to --cpu-vars variables); its ranges equal the
               device's when every end is exact (at the node limit a witnessed end depends on the width)
  naive ms     2n separate Solve() calls (presolve off) of the model with its objective turned into a bound row and
               +-one variable as the objective; their values must agree with the variable ranges when every end is
               exact

GPU name, power limit and clocks are read in the same run.  Usage: python scripts/mip_variability_bench.py [--runs 3]"""
from __future__ import annotations

import argparse
import json
import math
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
    bundle = {f["file"]: f["model"] for f in load_bundle()["fixtures"]}
    return [("Knapsack 1", bundle["Knapsack 1.json"]),
            ("knapsack 40", problems.single_knapsack_model(40, seed=3)),
            ("knapsack 40x5", problems.knapsack_mip_model(40, 5, seed=3)),
            ("random MIP 30x20", problems.random_mip_model(30, 20, seed=17, integer_fraction=0.5)),
            ("mixed MIP 60x40", problems.random_mip_model(60, 40, seed=29, integer_fraction=0.5)),
            ("Sudoku4x4", bundle["Sudoku4x4.json"])]


def naive(jm: dict, z: float, t: float):
    """({variable: (min, max)}, seconds) from 2n Solve() calls: the objective as a bound row, +-variable as objective."""
    import jslpsolver_b200 as J
    is_max = jm.get("opType") == "max"
    obj = jm.get("optimize")  # None: a feasibility model (Sudoku), every plan is optimal
    slack = 1e-9 * max(1.0, abs(z))
    cons = dict(jm["constraints"])
    if obj is not None:
        cons["__objective"] = {"min": z - t - slack} if is_max else {"max": z + t + slack}
    out, t0 = {}, time.perf_counter()
    for v in jm["variables"]:
        ends = []
        for sense in ("min", "max"):
            variables = {u: {**{k: x for k, x in spec.items() if k != obj}, "__objective": spec.get(obj, 0.0),
                             **({"__target": 1.0} if u == v else {})} for u, spec in jm["variables"].items()}
            m = dict(jm, constraints=cons, variables=variables, optimize="__target", opType=sense,
                     options={**(jm.get("options") or {}), "presolve": False})
            r = J.Solve(m)
            ends.append(r["result"] if r["bounded"] else (math.inf if sense == "max" else -math.inf))
        out[v] = tuple(ends)
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--max-nodes", type=int, default=20000)
    ap.add_argument("--width", type=int, default=None)
    ap.add_argument("--cpu-vars", type=int, default=50, help="run the restatement up to this many variables")
    ap.add_argument("--only", default=None, help="run the workloads whose name contains this")
    args = ap.parse_args()
    import jslpsolver_b200 as J
    import mip_variability_oracle as MO
    from oracle import ref_model
    from pool_bench import gpu_info
    from jslpsolver_b200.tableau import default_context
    ref_model.build_oracle()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name, jm in workloads():
        if args.only and args.only not in name:
            continue
        for gap in (0.0, 0.01):
            kw = dict(gap=gap, max_nodes=args.max_nodes, width=args.width)
            try:
                J.Variability(jm, **kw)  # warm-up
            except ValueError as e:
                print(json.dumps({"workload": name, "gap": gap, "refused": str(e)}), flush=True)
                continue
            best, r = None, None
            for _ in range(args.runs):
                default_context().sync()
                t0 = time.perf_counter()
                r = J.Variability(jm, **kw)
                dt = time.perf_counter() - t0
                best = dt if best is None else min(best, dt)
            cpu, same = None, None
            if len(jm["variables"]) <= args.cpu_vars:  # the restatement of the 60x40 MIP takes minutes
                t0 = time.perf_counter()
                o = MO.variability(jm, gap=gap, max_nodes=args.max_nodes, width=args.width)
                cpu = time.perf_counter() - t0
                same = {k: (e["min"], e["max"]) for k, e in r["variables"].items()} == \
                    {k: (e["min"], e["max"]) for k, e in o["variables"].items()}
            ranges, naive_s = naive(jm, r["optimum"], r["allowance"])
            scale = max(1.0, max(abs(x) for pair in ranges.values() for x in pair if math.isfinite(x)))
            agree = all(
                a is not None and ((a == b) if math.isinf(b) else abs(a - b) <= 1e-6 * scale)
                for v, pair in ranges.items() for a, b in zip((r["variables"][v]["min"], r["variables"][v]["max"]),
                                                               pair))
            # an end that reached --max-nodes holds the value its search witnessed, which depends on the width
            assert agree or not r["exact"], (name, gap, "the naive ranges disagree")
            print(json.dumps({"workload": name, "gap": gap, "exact": r["exact"], "searches": r["searches"],
                              "ms_per_call": round(1e3 * best, 2), "lps": r["lps"], "nodes": r["nodes"],
                              "lps_per_s": round(r["lps"] / best), "launches": r["launches"], "rounds": r["rounds"],
                              "pivots_per_lp": round(r["pivots"] / r["lps"], 1), "cpu_ms": None if cpu is None else round(1e3 * cpu, 2),
                              "naive_ms": round(1e3 * naive_s, 2), "same_ranges_as_restatement": same,
                              "naive_agrees": agree}), flush=True)


if __name__ == "__main__":
    main()

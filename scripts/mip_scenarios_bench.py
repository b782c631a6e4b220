"""Scenarios() on the device against a loop of Solve(edited_k) in the same process, alternated ABBA.  Workloads:
LargeFarmMIP with 64 and 512 right-hand-side perturbations, a 40x5 knapsack_mip_model with 256 cases and a 30x20
random_mip_model with 1024 cases.  Per workload and arm, every run:

  ms/call        host clock around the call (it ends in a device synchronise)
  trees/s        cases over the call time
  launches       kernel launches of the call
  node LPs       node LPs of the Scenarios() call, final re-solves included;  committed  the nodes its trees committed;
                 wasted  node LPs evaluated speculatively and never committed

Results of the two arms are checked equal.  GPU name and power limit are read in the same run.
Usage: python scripts/mip_scenarios_bench.py [--runs 2] [--cases N] [--only SUBSTRING,...]"""
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


def workloads(cap: int, only: str):
    from conftest import load_bundle
    from jslpsolver_b200 import problems
    from helpers import strip_timeouts
    from test_mip_scenarios_cpu import seeded_cases
    farm = strip_timeouts(next(f["model"] for f in load_bundle()["fixtures"] if f["file"] == "LargeFarmMIP.json"))
    rhs_only = lambda cases: [{"rhs": c["rhs"]} for c in cases]  # noqa: E731
    knap, rnd = problems.knapsack_mip_model(40, 5, seed=3), problems.random_mip_model(30, 20, seed=17)
    w = [("LargeFarmMIP", farm, rhs_only(seeded_cases(farm, 64, seed=1, spread=0.1))),
         ("LargeFarmMIP", farm, rhs_only(seeded_cases(farm, 512, seed=2, spread=0.1))),
         ("knapsack 40x5", knap, seeded_cases(knap, 256, seed=3)),
         ("random MIP 30x20", rnd, seeded_cases(rnd, 1024, seed=4))]
    keep = [x for x in only.split(",") if x]
    w = [(n, m, c[:cap] if cap else c) for n, m, c in w if not keep or any(k in n for k in keep)]
    return [(f"{n} x{len(c)}", m, c) for n, m, c in w]


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # reported, never guessed
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--cases", type=int, default=0, help="at most this many cases per workload (0 = all)")
    ap.add_argument("--only", default="", help="comma-separated substrings of the workload names to run")
    a = ap.parse_args()
    import jslpsolver_b200 as J
    from jslpsolver_b200 import mip_scenarios as MS
    from jslpsolver_b200.model import Model
    from jslpsolver_b200.tableau import default_context
    ctx = default_context()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name, jm, cases in workloads(a.cases, a.only):
        base = Model().loadJson(dict(jm, options={"presolve": False}))
        edited = [MS.edited(jm, base, c) for c in cases]
        s = J.Solver()

        def batch():
            l0 = ctx.launches
            t0 = time.perf_counter()
            out = s.Scenarios(jm, cases)
            return out, time.perf_counter() - t0, ctx.launches - l0

        def loop():
            l0 = ctx.launches
            t0 = time.perf_counter()
            out = [s.Solve(e) for e in edited]
            return out, time.perf_counter() - t0, ctx.launches - l0

        batch(), loop()  # warm-up of every shape
        rows = {"batch": [], "loop": []}
        for r in range(a.runs):
            for arm in (("batch", "loop") if r % 2 == 0 else ("loop", "batch")):
                out, sec, launches = (batch if arm == "batch" else loop)()
                rows[arm].append((sec, launches))
                print(json.dumps({"workload": name, "run": r, "arm": arm, "ms": round(1e3 * sec, 2)}), flush=True)
                if arm == "batch":
                    got = out
                else:
                    want = out
            assert got == want, name
        for arm, v in rows.items():
            ms = [1e3 * x for x, _ in v]
            print(json.dumps({"workload": name, "arm": arm, "cases": len(cases), "ms": [round(x, 2) for x in ms],
                              "trees_per_s": round(len(cases) / (min(ms) / 1e3), 1), "launches": v[0][1]}),
                  flush=True)
        # counters of one call, from the C status records
        inst = s._instance(dict(jm, options={"presolve": False}), None)
        col0, row0 = zip(*[MS.edges(inst.initial_tableau(), Model().loadJson(e).initial_tableau()) for e in edited])
        tab = inst.tableau
        tab.setModel(inst)
        st = tab.bnb_batch(list(col0), list(row0), tolerance=float(inst.tolerance or 0))
        tab.close()
        lps = sum(x.nodes_evaluated for x in st["status"])
        committed = sum(x.iterations for x in st["status"])
        print(json.dumps({"workload": name, "node_lps": lps, "committed": committed,
                          "wasted": lps - committed - sum(1 for x in st["status"] if x.iterations > 1),
                          "launches": st["launches"]}), flush=True)


if __name__ == "__main__":
    main()

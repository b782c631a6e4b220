"""FrontierMIP() on the device against the sequential restatement (tests/frontier_mip_oracle.py, on the CPU) and against
what a user writes without it: an epsilon-constraint loop of Solve() calls on edited JSON models (from eps = inf:
minimise g1 under g2 <= eps, then g2 under g1 <= that optimum and g2 <= eps, then eps = g2 - 1; presolve off).
Workloads: seeded bi-objective 0/1 knapsacks and assignment models (tests/test_frontier_mip_cpu.py) with conflicting
objectives, 5 to 100+ frontier points.  The three ways run alternated, once each per run, --runs times after one warm-up.  Per workload:

  points       frontier points;  ms  host clock around the call (each ends in a device synchronise), best of --runs
  launches     device launches of one FrontierMIP() call;  searches, lps, nodes, rounds, pivots its counters
  boxes        live boxes of every stage;  launches/wave  launches of the box stages over their waves (rounds)
  cpu ms       the restatement at the device's width; "same" says its result equals the device's
  solve ms     the epsilon-constraint loop; "agrees" says its images equal the device's within 1e-6

GPU name, power limit and clocks are read in the same run.  Usage: python scripts/frontier_mip_bench.py [--runs 3]"""
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

WIDTH = 16


def conflicting(jm: dict, a: str, b: str, top: int) -> dict:
    """jm with objective b set to top - a (plus 0..2) on every variable: the two objectives pull apart, so the frontier
    has many points."""
    import numpy as np
    rng = np.random.default_rng(len(jm["variables"]))
    return dict(jm, variables={v: dict(c, **{b: top - c[a] + int(rng.integers(0, 3))}) for v, c in jm["variables"].items()})


def workloads():
    from test_frontier_mip_cpu import assignment, knapsack
    return [(f"knapsack {n}", conflicting(knapsack(n, 11), "p1", "p2", 30)) for n in (10, 16, 20)] + \
        [(f"assignment {n}x{n}", conflicting(assignment(n, 11), "cost", "time", 20)) for n in (4, 6, 8, 10)]


def by_solve(jm: dict) -> list:
    """The images (g1, g2) of the epsilon-constraint loop, two Solve() calls per point."""
    import jslpsolver_b200 as J
    from jslpsolver_b200.frontier import _coef
    from jslpsolver_b200.model import object_keys
    keys = object_keys(jm["optimize"])
    sig = {k: 1.0 if jm["optimize"][k] == "min" else -1.0 for k in keys}
    g = {vid: [sig[k] * _coef(jm, vid, k) for k in keys] for vid in jm["variables"]}
    variables = {vid: dict({a: x for a, x in spec.items() if a not in keys}, __g1=g[vid][0], __g2=g[vid][1],
                            __c1=g[vid][0], __c2=g[vid][1]) for vid, spec in jm["variables"].items()}
    base = dict(jm, variables=variables, options={"presolve": False})
    out, eps = [], None

    def image(sol):
        return tuple(sum(g[v][i] * sol.get(v, 0.0) for v in jm["variables"]) for i in (0, 1))

    while True:
        rows = dict(jm["constraints"], **({} if eps is None else {"__c2": {"max": eps}}))
        s1 = J.Solve(dict(base, constraints=rows, optimize="__g1", opType="min"))
        if not s1["feasible"]:
            return out
        v1 = image(s1)[0]
        s2 = J.Solve(dict(base, constraints=dict(rows, __c1={"max": v1 + 1e-9 * max(1.0, abs(v1))}),
                          optimize="__g2", opType="min"))
        img = image(s2)
        out.append(img)
        eps = img[1] - 1.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    import jslpsolver_b200 as J
    import frontier_mip_oracle as FO
    from jslpsolver_b200 import frontier_mip as FM
    from jslpsolver_b200.tableau import default_context
    from oracle import ref_model
    from pool_bench import gpu_info
    from test_frontier_mip_cpu import images
    ref_model.build_oracle()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    stages, run = [], FM.run

    def logged(evaluate, targets, *a, **k):  # live boxes and launches / waves of every box stage
        l0 = default_context().launches
        out = run(evaluate, targets, *a, **k)
        stages.append((len(targets), default_context().launches - l0, out["rounds"]))
        return out

    FM.run = logged
    for name, jm in workloads():
        r = J.FrontierMIP(jm, width=WIDTH)  # warm-up
        naive = by_solve(jm)
        best = {"device": None, "cpu": None, "solve": None}
        for _ in range(args.runs):
            stages.clear()
            default_context().sync()
            t0 = time.perf_counter()
            r = J.FrontierMIP(jm, width=WIDTH)
            t1 = time.perf_counter()
            o, _ = FO.frontier_mip(jm, width=WIDTH)
            t2 = time.perf_counter()
            naive = by_solve(jm)
            default_context().sync()
            t3 = time.perf_counter()
            for k, dt in (("device", t1 - t0), ("cpu", t2 - t1), ("solve", t3 - t2)):
                best[k] = dt if best[k] is None else min(best[k], dt)
        same = all(r[k] == o[k] for k in o)
        got = images(r["points"], jm)
        agrees = len(got) == len(naive) and all(abs(a - b) <= 1e-6 for p, q in zip(got, naive) for a, b in zip(p, q))
        box = [s for s in stages if s[0] > 0]
        print(json.dumps({"workload": name, "stop": r["stop"], "points": len(r["points"]),
                          "ms": round(1e3 * best["device"], 2), "launches": r["launches"], "searches": r["searches"],
                          "lps": r["lps"], "nodes": r["nodes"], "rounds": r["rounds"], "pivots": r["pivots"],
                          "boxes": [s[0] for s in box],
                          "launches_per_wave": round(sum(s[1] for s in box) / max(1, sum(s[2] for s in box)), 2),
                          "cpu_ms": round(1e3 * best["cpu"], 2), "same": same,
                          "solve_ms": round(1e3 * best["solve"], 2), "agrees": agrees}), flush=True)


if __name__ == "__main__":
    main()

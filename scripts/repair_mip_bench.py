"""RepairMIP() on the device against the sequential restatement (tests/repair_mip_oracle.py, on the CPU) and against
what a user does without it: the elastic model written as JSON (one violation variable per row side, objective the
weighted violation) solved with Solve(), then the same model with the model's objective and the bound row
sum w e <= V* + t, solved with Solve() again (presolve off in both).  Workloads: seeded infeasible packing MIPs
(problems.infeasible_packing_model with every variable integer) and a planted parity conflict
(problems.planted_integer_conflict_model), every row relaxable with weight 1, at gap 0 and 0.01.  The three ways run
alternated, once each per run, --runs times after one warm-up.  Per workload and gap:

  ms           host clock around the call (each ends in a device synchronise or runs on the CPU), best of --runs
  launches     device launches of one RepairMIP() call;  lps, nodes, rounds, pivots its counters
  cpu ms       the restatement on the C oracle at the device's width (16); "same" says its result equals the device's
  solve ms     the two Solve() calls; "agrees" says V* and the result equal the device's within 1e-6 relative

GPU name, power limit and clocks are read in the same run.  Usage: python scripts/repair_mip_bench.py [--runs 3]"""
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


def workloads():
    from jslpsolver_b200 import problems

    def ints(jm):
        return dict(jm, ints={v: 1 for v in jm["variables"]})

    return [("packing MIP 20x16, 4 demand", ints(problems.infeasible_packing_model(20, 16, 4, seed=5))),
            ("packing MIP 30x24, 6 demand", ints(problems.infeasible_packing_model(30, 24, 6, seed=7))),
            ("planted parity 30x40, k=4", problems.planted_integer_conflict_model(30, 40, 4, seed=3))]


def by_solve(jm: dict, gap: float) -> tuple:
    """(V*, result) from two Solve() calls on the elastic model written as JSON: every constraint side is its own row
    with a violation variable, stage 1 minimises their sum, stage 2 optimises the model's objective under the bound
    row sum e <= V* + t (widened by 1e-9 relative, as the solver meets rows within its precision)."""
    import jslpsolver_b200 as J
    rows, variables, viol = {}, {v: dict(spec) for v, spec in jm["variables"].items()}, []
    for name, spec in jm["constraints"].items():
        sides = [("min", spec["equal"]), ("max", spec["equal"])] if spec.get("equal") is not None else \
            [(s, spec[s]) for s in ("min", "max") if spec.get(s) is not None]
        for side, rhs in sides:
            row, e = f"{name}__{side}", f"__e_{name}_{side}"
            rows[row] = {side: rhs}
            for v, coefs in jm["variables"].items():
                if name in coefs:
                    variables[v][row] = coefs[name]
            variables[e] = {row: 1.0 if side == "min" else -1.0, "__violation": 1.0}
            viol.append(e)
    for v, coefs in variables.items():
        for name in jm["constraints"]:
            coefs.pop(name, None)
    base = dict(jm, constraints=rows, variables=variables, options={"presolve": False})
    s1 = J.Solve(dict(base, optimize="__violation", opType="min"))
    vstar = s1["result"]
    cap = vstar + gap * abs(vstar)
    rows2 = dict(rows, __bound={"max": cap + 1e-9 * max(1.0, cap)})
    s2 = J.Solve(dict(base, constraints=rows2, variables={v: dict(c, __bound=c.get("__violation", 0.0))
                                                          for v, c in variables.items()}))
    return vstar, s2.get("result")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    import jslpsolver_b200 as J
    import repair_mip_oracle as RMO
    from oracle import ref_model
    from pool_bench import gpu_info
    from jslpsolver_b200.tableau import default_context
    ref_model.build_oracle()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name, jm in workloads():
        for gap in (0.0, 0.01):
            r = J.RepairMIP(jm, gap=gap, width=WIDTH)  # warm-up
            by_solve(jm, gap)
            best = {"device": None, "cpu": None, "solve": None}
            for _ in range(args.runs):
                default_context().sync()
                t0 = time.perf_counter()
                r = J.RepairMIP(jm, gap=gap, width=WIDTH)
                t1 = time.perf_counter()
                o, _ = RMO.repair_mip(jm, gap=gap, width=WIDTH)
                t2 = time.perf_counter()
                naive = by_solve(jm, gap)
                default_context().sync()
                t3 = time.perf_counter()
                for k, dt in (("device", t1 - t0), ("cpu", t2 - t1), ("solve", t3 - t2)):
                    best[k] = dt if best[k] is None else min(best[k], dt)
            same = all(r[k] == o[k] for k in o)
            vstar = r["stages"][0]["optimum"]
            agrees = naive[1] is not None and all(abs(a - b) <= 1e-6 * max(1.0, abs(a), abs(b))
                                                  for a, b in zip((vstar, r["result"]), naive))
            print(json.dumps({"workload": name, "gap": gap, "stop": r["stop"], "violation": r["violation"],
                              "result": r["result"], "tableau": [(s["height"], s["width"]) for s in r["stages"]],
                              "ms": round(1e3 * best["device"], 2), "launches": r["launches"], "lps": r["lps"],
                              "nodes": r["nodes"], "rounds": r["rounds"], "pivots": r["pivots"],
                              "cpu_ms": round(1e3 * best["cpu"], 2), "same": same,
                              "solve_ms": round(1e3 * best["solve"], 2), "solve": naive, "agrees": agrees}),
                  flush=True)


if __name__ == "__main__":
    main()

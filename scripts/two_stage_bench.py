"""Two-stage stochastic LPs (DESIGN.md section 2u): TwoStage() on seeded capacity-expansion models at S = 64, 256 and
1024 cases, against the same L-shaped loop with the recourse LPs solved one case at a time on the CPU (the restatement
over the C oracle, tests/two_stage_oracle.py) and against Solve() of the deterministic equivalent while it fits the
tableau's width cap.  Prints one JSON line per S.  Run from the repository root on a GPU machine:

    python scripts/two_stage_bench.py [--cases 64 256 1024] [--no-cpu]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

WIDTH_CAP = 25600  # dense tableau columns (DESIGN.md section 7)


def equivalent(model, cases, first, p):
    """The deterministic equivalent as one JSON model: every second-stage row and variable copied per case."""
    variables, constraints, obj = model["variables"], model["constraints"], model["optimize"]
    second = [v for v in variables if v not in first]
    srows = [n for n in constraints if any(variables[y].get(n, 0) for y in second)]
    total = sum(p)
    cons = {n: dict(c) for n, c in constraints.items() if n not in srows}
    out = {x: {k: v for k, v in variables[x].items() if k not in srows} for x in first}
    for s, case in enumerate(cases):
        for n in srows:
            spec = dict(constraints[n])
            r = (case.get("rhs") or {}).get(n)
            if r is not None:
                spec = {k: r for k in spec}
            cons[f"{n}@{s}"] = spec
            for x in first:
                t = (case.get("coefficients") or {}).get(n, {}).get(x, variables[x].get(n, 0))
                if t:
                    out[x][f"{n}@{s}"] = t
        for y in second:
            cost = (case.get("cost") or {}).get(y, variables[y].get(obj, 0))
            out[f"{y}@{s}"] = {obj: p[s] / total * cost, **{f"{n}@{s}": variables[y][n] for n in srows if n in variables[y]}}
    return {"optimize": obj, "opType": model.get("opType", "min"), "constraints": cons, "variables": out,
            "options": {"presolve": False}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, nargs="+", default=[64, 256, 1024])
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    import subprocess
    import two_stage_models as TM
    import two_stage_oracle as TO
    import jslpsolver_b200 as J
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    for S in args.cases:
        model, cases, first, p = TM.capacity(11, n_first=10, n_second=30, n_cases=S, per_case_t=True)
        J.TwoStage(model, cases[:4], first, p[:4])  # warm-up: module load and kernel attributes
        t0 = time.perf_counter()
        r = J.TwoStage(model, cases, first, p)
        t_gpu = time.perf_counter() - t0
        row = {"S": S, "gpu": gpu, "iterations": len(r["iterations"]), "stop": r["stop"], "result": r["result"],
               "recourse_lps": r["recourse_lps"], "pivots": r["pivots"], "launches": r["launches"],
               "two_stage_s": round(t_gpu, 4)}
        if not args.no_cpu:
            t0 = time.perf_counter()
            o = TO.TwoStage(model, cases, first, p)
            row["cpu_restatement_s"] = round(time.perf_counter() - t0, 4)
            row["same_as_restatement"] = o["result"] == r["result"] and o["first"] == r["first"]
        de = equivalent(model, cases, first, p)
        width = 1 + len(de["variables"])
        row["equivalent_width"] = width
        if width <= WIDTH_CAP:
            t0 = time.perf_counter()
            d = J.Solve(de)
            row["equivalent_solve_s"] = round(time.perf_counter() - t0, 4)
            row["equivalent_result"] = d["result"]
        else:
            row["equivalent_solve_s"] = None  # beyond the tableau's width cap: no single-model answer
        print(json.dumps(row), flush=True)
    # the smallest S whose deterministic equivalent no longer fits the width cap
    model, cases, first, p = TM.capacity(11, n_first=10, n_second=30, n_cases=1, per_case_t=True)
    per_case = len(equivalent(model, cases, first, p)["variables"]) - len(first)
    print(json.dumps({"equivalent_exceeds_width_cap_at_S": (WIDTH_CAP - 1 - len(first)) // per_case + 1}))


if __name__ == "__main__":
    main()

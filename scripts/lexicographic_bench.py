"""Time lexicographic objectives on one GPU: each level of the warm chain (jslp_lex_next, then a phase 2 on the new
tableau) against the cold chain a user writes without it (one Solve() per level, the earlier objectives added to the
JSON model as constraints `objective_j >= z_j - t_j` for max or `<= z_j + t_j` for min).

For each model and gap, after one warm-up of both chains, each chain runs twice.  Per level the warm chain records the
time to build the next tableau (host clock around jslp_lex_next, which ends in a stream synchronise), its phase-2
pivots and the level time (build plus simplex, or Solve() for level 1); the cold chain records the Solve() time of
each level.  "optima_agree" says whether both chains reached the same level optima to 1e-6 relative (a cold Solve()
can end "infeasible" when its bound row is tight, and the chain then stops there; a warm level after a face that
keeps only the optimum runs no LP and has no optimum of its own here).  Prints one JSON line per model and gap
with the device name and power limit read in the same run.

    python scripts/lexicographic_bench.py [--sizes 150x120,550x600,2000x2000] [--gaps 0,0.01] [--objectives 3]
"""
from __future__ import annotations

import argparse
import json
import os
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


def warm_chain(jm, gap):
    """The levels of Lexicographic(jm, gap) on the tableau API, timed: [{"optimum", "kind", "build_ms", "pivots",
    "level_ms"}], total ms."""
    import jslpsolver_b200 as J
    from jslpsolver_b200.frontier import cost_row
    keys = list(jm["optimize"])
    senses = jm["optimize"]
    working = dict(jm, optimize=keys[0], opType=senses[keys[0]])
    t_all = time.perf_counter()
    inst = J.solver._instance(working, None)
    sol = inst.solve()
    assert sol.feasible and sol.bounded
    cur = inst.tableau
    st = cur.lastStatus
    z = -(1.0 if senses[keys[0]] == "max" else -1.0) * float(cur.cost_row()[0])
    levels = [{"optimum": z, "kind": "solve", "build_ms": 0.0, "pivots": st.phase1_pivots + st.phase2_pivots,
               "level_ms": (time.perf_counter() - t_all) * 1e3}]
    for key in keys[1:]:
        t0 = time.perf_counter()
        t = gap * abs(z)
        nxt, _ = cur.lex_next(cost_row(inst, working, key, senses[key], cur.nVars), t)
        build = (time.perf_counter() - t0) * 1e3
        if cur is not inst.tableau:
            cur.close()
        cur = nxt
        if cur is None:  # a face that keeps only the optimum: the later levels run no LP
            levels.append({"optimum": None, "kind": None, "build_ms": build, "pivots": 0, "level_ms": build})
            break
        cur.simplex(check_cycles=True)
        assert cur.feasible and cur.bounded and cur.lastStatus.phase1_pivots == 0
        z = -(1.0 if senses[key] == "max" else -1.0) * float(cur.cost_row()[0])
        levels.append({"optimum": z, "kind": "face" if t == 0.0 else "bound", "build_ms": build,
                       "pivots": cur.lastStatus.phase2_pivots, "level_ms": (time.perf_counter() - t0) * 1e3})
    if cur is not None and cur is not inst.tableau:
        cur.close()
    return levels, (time.perf_counter() - t_all) * 1e3


def cold_chain(jm, gap):
    """The same levels as cold Solve() calls with the earlier objectives as JSON constraints: [{"optimum", "ms"}],
    total ms."""
    import jslpsolver_b200 as J
    keys = list(jm["optimize"])
    senses = jm["optimize"]
    base = {k: v for k, v in jm.items() if k != "optimize"}
    levels, cons, variables = [], dict(jm["constraints"]), {v: dict(a) for v, a in jm["variables"].items()}
    t_all = time.perf_counter()
    for k, key in enumerate(keys):
        model = dict(base, optimize=key, opType=senses[key], constraints=dict(cons), variables=variables)
        t0 = time.perf_counter()
        res = J.Solve(model)
        ms = (time.perf_counter() - t0) * 1e3
        if not (res["feasible"] and res["bounded"]):  # a cold start can end "infeasible" on an equality-tight bound
            levels.append({"optimum": None, "ms": ms, "feasible": res["feasible"], "bounded": res["bounded"]})
            break
        z = float(res["result"])
        levels.append({"optimum": z, "ms": ms})
        t = gap * abs(z)
        name = f"__level{k}"
        cons[name] = {"min": z - t} if senses[key] == "max" else {"max": z + t}
        for vid, attrs in variables.items():
            if attrs.get(key):
                attrs[name] = attrs[key]
    return levels, (time.perf_counter() - t_all) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="150x120,550x600,2000x2000")
    ap.add_argument("--gaps", default="0,0.01")
    ap.add_argument("--objectives", type=int, default=3)
    ap.add_argument("--seed", type=int, default=12345)
    args = ap.parse_args()
    import torch
    from jslpsolver_b200 import problems
    dev, cond = torch.cuda.get_device_name(0), gpu_conditions()
    for size in args.sizes.split(","):
        n_vars, n_cons = (int(x) for x in size.split("x"))
        for family, make in (("alternative_optima_multi", problems.alternative_optima_multi_model),
                             ("dense_packing_multi", problems.dense_packing_multi_model)):
            jm = make(n_vars, n_cons, args.objectives, seed=args.seed)
            for gap in (float(g) for g in args.gaps.split(",")):
                warm_chain(jm, gap)  # warm-up: module load, first launches, buffers of this shape
                cold_chain(jm, gap)
                runs = []
                for _ in range(2):
                    wl, wt = warm_chain(jm, gap)
                    cl, ct = cold_chain(jm, gap)
                    agree = all(
                        a["optimum"] is None or (b["optimum"] is not None and
                                                 abs(a["optimum"] - b["optimum"]) <= 1e-6 * max(1.0, abs(b["optimum"])))
                        for a, b in zip(wl, cl))
                    runs.append({"warm": {"levels": wl, "total_ms": wt}, "cold": {"levels": cl, "total_ms": ct},
                                 "optima_agree": agree})
                print(json.dumps({"device": dev, **cond, "family": family, "tableau": f"{n_cons + 1}x{n_vars + 1}",
                                  "objectives": args.objectives, "gap": gap, "runs": runs}), flush=True)


if __name__ == "__main__":
    main()

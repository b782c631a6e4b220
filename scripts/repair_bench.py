"""Repair() on the device at three sizes of problems.infeasible_packing_model (a quarter of the rows are demand rows
that make the model infeasible; every row may be relaxed).  Per size and run:

  build      jslp_elastic_create (the elastic tableau, crash included) against the same tableau built on the host
             without the crash, uploaded, and crashed by jslp_crash onto the same rows (one pivot per crashed row)
  stage 1/2  simplex() of the violation LP and of the re-optimised objective over the plans within 1 % of V*
             (jslp_lex_next + simplex()), with pivots
  cold       what a user writes today: the elastic model as JSON through two cold Solve() calls, the second with the
             total violation capped at V* (skipped with --no-cold and at the largest size by default)

GPU name, power limit and clocks are read in the same run.  Usage: python scripts/repair_bench.py [--runs 2]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = [(120, 150), (600, 550), (2000, 2000)]  # (rows, variables): tableaux 121x151, 601x551, 2001x2001


def gpu_info() -> str:
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def timed(fn):
    from jslpsolver_b200.tableau import default_context
    default_context().sync()
    t0 = time.perf_counter()
    out = fn()
    default_context().sync()
    return out, 1e3 * (time.perf_counter() - t0)


def host_elastic(it, rows, w):
    """The elastic tableau before the crash, built on the host: row 0 = -w at every elastic column."""
    M = it.matrix
    H, W = M.shape
    E = np.zeros((H, W + len(rows)))
    E[:, :W] = M
    E[0, :W] = 0.0
    for j, r in enumerate(rows):
        E[r, W + j] = -1.0
        E[0, W + j] = -w[j]
    vcol = np.concatenate([it.varIndexByCol, H + W - 2 + np.arange(len(rows))]).astype(np.int32)
    return E, it.varIndexByRow, vcol


def elastic_json(A, b, lower, c, vstar=None):
    """The user's elastic model: one e_i per row, minimise sum e (or, with vstar, maximise c.x with sum e <= vstar)."""
    from jslpsolver_b200 import problems
    jm = problems.lp_model(A, b, c, lower)
    n = len(b)
    for i in range(n):
        jm["variables"][f"e{i}"] = {f"c{i}": (1.0 if lower[i] else -1.0), "violation": 1.0,
                                    "objective": 0.0}
    if vstar is None:
        return dict(jm, optimize="violation", opType="min")
    jm["constraints"]["violation"] = {"max": vstar}
    return jm


def run(n_cons, n_vars, cold):
    from jslpsolver_b200 import problems
    from jslpsolver_b200.repair import objective_row
    from jslpsolver_b200.tableau import GpuTableau
    import jslpsolver_b200 as J
    A, b, c, lower = problems.infeasible_packing_arrays(n_vars, n_cons, n_cons // 4, seed=1)
    it = problems.lp_tableau(A, b, c, lower)
    H, W = it.matrix.shape
    rows, w = list(range(1, H)), [1.0] * (H - 1)
    out = {"size": f"{H}x{W}", "crashed_rows": int(lower.sum())}
    g = GpuTableau(1e-8)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol)
    (e, n), out["build_ms"] = timed(lambda: g.elastic(rows, w))
    out["crashed"] = n
    # the same tableau from the host, crashed by jslp_crash (one rank-1 pivot per crashed row)
    E0, vr, vc = host_elastic(it, rows, w)
    h = GpuTableau(1e-8)

    def host_path():
        h.upload(E0, vr, vc, row_capacity=H + 1)
        crashed = [j for j, r in enumerate(rows) if it.matrix[r, 0] < -1e-8]
        leave = np.zeros(h.nVars, dtype=np.uint8)
        leave[[int(it.varIndexByRow[rows[j]]) for j in crashed]] = 1
        return h.crash([H + W - 2 + j for j in crashed], leave)

    (_, pivots), out["host_crash_ms"] = timed(host_path)
    out["host_crash_pivots"] = pivots
    h.close()
    g.close()
    _, out["stage1_ms"] = timed(lambda: e.simplex(check_cycles=True))
    st = e.lastStatus
    out["stage1_pivots"] = [int(st.phase1_pivots), int(st.phase2_pivots)]
    out["vstar"] = float(e.cost_row()[0])
    t = 0.01 * out["vstar"]
    (nxt, _), out["stage2_build_ms"] = timed(lambda: e.lex_next(objective_row(it, e.nVars), t))
    if nxt is not None:
        _, out["stage2_ms"] = timed(lambda: nxt.simplex(check_cycles=True))
        out["stage2_pivots"] = int(nxt.lastStatus.phase2_pivots)
        out["result"] = -float(nxt.cost_row()[0])
        nxt.close()
    e.close()
    if cold:
        t0 = time.perf_counter()
        first = J.Solve(elastic_json(A, b, lower, c))
        second = J.Solve(elastic_json(A, b, lower, c, first["result"] if first["feasible"] else 0.0))
        out["cold_ms"] = 1e3 * (time.perf_counter() - t0)
        out["cold"] = [first.get("result"), second.get("result"), bool(second.get("feasible"))]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--no-cold", action="store_true")
    ap.add_argument("--cold-max-rows", type=int, default=600)
    ap.add_argument("--sizes", default="0,1,2", help="indices into SIZES")
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for n_cons, n_vars in [SIZES[int(i)] for i in args.sizes.split(",")]:
        for k in range(args.runs):
            out = run(n_cons, n_vars, not args.no_cold and n_cons <= args.cold_max_rows)
            out["run"] = k + 1
            print(json.dumps(out), flush=True)
    print(json.dumps({"gpu": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()

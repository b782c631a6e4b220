"""Time the warm start on one GPU: a cold solve against a warm start from the optimal basis of the unedited LP.

For each size, solves a seeded dense packing LP (bench.py's generator), takes its optimal basis, applies one edit
(same = none, coef = every coefficient x (1 + 0.02 N(0,1)), rhs = every right-hand side x (1 + 0.1 N(0,1)), cost =
every cost x (1 + 0.1 N(0,1)), rows = 1 % more rows) and times two arms, alternated, each on the host clock around
work that ends in a synchronise:
  LP phase      cold: upload, simplex(), read-back of column 0      warm: upload, jslp_crash, simplex(), read-back
  whole Solve   Solve(model) against Solve(model, basis=...) on the JSON model (model build and presolve included;
                sizes up to --solve-max-vars only: the Python model build of the largest LP dominates and is slow)
Reports the pivots of each arm, the crash time and its time per crash pivot, and whether the objectives agree to
1e-9 relative.  Prints one JSON line per case with the device name and power limit beside the numbers.

    python scripts/warmstart_bench.py [--sizes 150x120,550x600,2000x2000] [--edits same,coef,rhs,cost,rows] [--reps 3]
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


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", os.environ.get("JSLP_DEVICE", "0"), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def edited(A, b, c, edit, rng):
    import numpy as np
    A2, b2, c2 = A.copy(), b.copy(), c.copy()
    if edit == "coef":
        A2 *= 1 + 0.02 * rng.standard_normal(A.shape)
    elif edit == "rhs":
        b2 *= 1 + 0.1 * rng.standard_normal(b.shape)
    elif edit == "cost":
        c2 *= 1 + 0.1 * rng.standard_normal(c.shape)
    elif edit == "rows":
        k = max(2, len(b) // 100)
        A2 = np.vstack([A, rng.integers(1, 21, size=(k, A.shape[1])).astype(float)])
        b2 = np.concatenate([b, rng.integers(100, 301, size=k).astype(float)])
    elif edit != "same":
        raise SystemExit(f"unknown edit {edit!r}")
    return A2, b2, c2


def lp_phase(it, ctx, enter=None, leave=None):
    """(ms, crash ms, crash pivots, p1, p2, raw objective) of one upload [+ crash] + simplex + read-back."""
    from jslpsolver_b200.tableau import GpuTableau
    t0 = time.perf_counter()
    g = GpuTableau(1e-8, context=ctx)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol)
    crash_ms, n = 0.0, 0
    if enter is not None:
        ctx.sync()
        t1 = time.perf_counter()
        _, n = g.crash(enter, leave)
        crash_ms = (time.perf_counter() - t1) * 1e3
    g.simplex()
    raw = float(g.rhs_column()[0])
    ms = (time.perf_counter() - t0) * 1e3
    st = g.lastStatus
    out = (ms, crash_ms, n, st.phase1_pivots, st.phase2_pivots, raw, bool(st.feasible and st.bounded))
    g.close()
    return out


def run_case(nv, nc, edit, seed, reps, whole):
    import numpy as np
    import jslpsolver_b200 as J
    from jslpsolver_b200 import problems
    from jslpsolver_b200.tableau import GpuTableau, default_context
    ctx = default_context()
    A, b, c = problems.dense_packing_lp_arrays(nv, nc, seed)
    it0 = problems.lp_tableau(A, b, c)
    g = GpuTableau(1e-8, context=ctx)
    g.upload(it0.matrix, it0.varIndexByRow, it0.varIndexByCol)
    g.simplex()
    vrow, vcol = np.array(g.varIndexByRow), np.array(g.varIndexByCol)
    g.close()
    var_labels = set(int(x) for x in it0.varIndexByCol[1:])
    A2, b2, c2 = edited(A, b, c, edit, np.random.default_rng(seed + 1))
    it = problems.lp_tableau(A2, b2, c2)
    n_labels = it.matrix.shape[0] + it.matrix.shape[1] - 2
    # the labels of the saved basis, as plan() resolves them on the edited model (rows first, then variables)
    shift = A2.shape[0] - A.shape[0]
    relabel = lambda x: int(x) + shift if int(x) in var_labels else int(x)
    enter = np.array([relabel(x) for x in vrow[1:] if int(x) in var_labels], dtype=np.int32)
    leave = np.zeros(n_labels, dtype=np.uint8)
    leave[[int(x) for x in vcol[1:] if int(x) not in var_labels]] = 1
    lp_phase(it, ctx), lp_phase(it, ctx, enter, leave)  # warm-up: kernel attributes, graphs
    cold, warm = [], []
    for _ in range(reps):  # alternated
        cold.append(lp_phase(it, ctx))
        warm.append(lp_phase(it, ctx, enter, leave))
    med = lambda xs, k: float(np.median([x[k] for x in xs]))
    c0, w0 = cold[0], warm[0]
    agree = c0[6] == w0[6] and (not c0[6] or abs(c0[5] - w0[5]) <= 1e-9 * max(1.0, abs(c0[5])))
    out = {"tableau": f"{it.matrix.shape[0]}x{it.matrix.shape[1]}", "edit": edit, "reps": reps,
           "cold_pivots": [c0[3], c0[4]], "warm_pivots": [w0[2], w0[3], w0[4]],
           "cold_lp_ms": med(cold, 0), "warm_lp_ms": med(warm, 0), "crash_ms": med(warm, 1),
           "crash_us_per_pivot": (1e3 * med(warm, 1) / w0[2]) if w0[2] else None,
           "objectives_agree_1e-9": bool(agree)}
    if whole:
        jm = problems.lp_model(A2, b2, c2)
        basis = J.Solve(problems.lp_model(A, b, c), full=True).basis()
        ts_c, ts_w, rc, rw = [], [], None, None
        for _ in range(reps):
            t0 = time.perf_counter()
            rc = J.Solve(jm)
            ts_c.append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter()
            rw = J.Solve(jm, basis=basis)
            ts_w.append((time.perf_counter() - t0) * 1e3)
        out.update({"cold_solve_ms": float(np.median(ts_c)), "warm_solve_ms": float(np.median(ts_w)),
                    "solve_results_agree_1e-9": abs(rc["result"] - rw["result"]) <= 1e-9 * max(1.0, abs(rc["result"]))})
    else:
        out.update(cold_solve_ms=None, warm_solve_ms=None, whole_solve="not measured at this size")
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="150x120,550x600,2000x2000", help="comma-separated VARSxCONS")
    ap.add_argument("--edits", default="same,coef,rhs,cost,rows")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--solve-max-vars", type=int, default=600)
    ap.add_argument("--seed", type=int, default=12345)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only measures on the GPU")
    dev, pw = torch.cuda.get_device_name(0), power_limit_w()
    for spec in a.sizes.split(","):
        nv, nc = (int(x) for x in spec.split("x"))
        for edit in a.edits.split(","):
            out = run_case(nv, nc, edit, a.seed, a.reps, nv <= a.solve_max_vars)
            out.update(device=dev, power_limit_w=pw)
            print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

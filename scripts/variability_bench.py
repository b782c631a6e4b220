"""Time the ranges of every variable and slack over the optimal face on one GPU: the device face (jslp_face_create) and
one scenario batch on it, against the way a user gets the same numbers without it.

For each size, solves a seeded LP with planted alternative optima (problems.alternative_optima_arrays) once, and lists
the targets of DESIGN.md section 2h rule 4 for every structural variable and every row.  Arms, each timed on the host
clock around work that ends in a synchronise, after one warm-up, the two alternated --reps times:
  device  GpuTableau.face() (face_ms), then one scenario_batch of all targets on the face (batch_ms)
  host    download the whole tableau, select the kept columns in NumPy, create and upload a new tableau
          (host_face_ms), then the same scenario_batch (host_batch_ms)
Checks that device and host agree bit for bit (kept columns, statuses, every final column 0).  The third way, one fresh
Solve() per target with an added `objective = z*` row, is not run here and is listed under "not_measured".  Prints one
JSON line per size with the device name, power limit and clocks beside the numbers.

    python scripts/variability_bench.py [--sizes 150x120,550x600,2000x2000] [--reps 5] [--seed 12345]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
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


def targets_of(vrow, vcol, kept):
    """Rule 4 for every label of the tableau: two LPs per basic label, one per non-basic label in a kept column."""
    t = []
    for lab in vrow[1:]:
        t += [(int(lab), -1), (int(lab), 1)]
    return t + [(int(vcol[c]), 1) for c in kept[1:]]


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def run_size(n_vars, n_cons, reps, seed):
    import numpy as np
    from jslpsolver_b200 import problems
    from jslpsolver_b200.tableau import GpuTableau
    A, b, c = problems.alternative_optima_arrays(n_vars, n_cons, seed)
    it = problems.lp_tableau(A, b, c)
    g = GpuTableau(1e-8)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol)
    t0 = time.perf_counter()
    g.simplex()
    solve_ms = (time.perf_counter() - t0) * 1e3
    assert g.feasible and g.bounded, "the benchmark LP has no optimum"
    H, W = g.height, g.width
    vrow, vcol = np.array(g.varIndexByRow), np.array(g.varIndexByCol)
    P = g.precision

    def device():
        t0 = time.perf_counter()
        f, kept = g.face()
        t1 = time.perf_counter()
        tg = targets_of(vrow, vcol, kept)
        out = f.scenario_batch([(1, lab, float(-s)) for lab, s in tg], list(range(len(tg) + 1)), check_cycles=True)
        t2 = time.perf_counter()
        f.close()
        return (t1 - t0) * 1e3, (t2 - t1) * 1e3, kept, tg, out

    def host():
        t0 = time.perf_counter()
        g._cache.clear()
        M = g.matrix2d()
        kept = np.concatenate([[0], 1 + np.nonzero((M[0, 1:] >= -P) & (M[0, 1:] <= P))[0]]).astype(np.int32)
        F = np.ascontiguousarray(M[:, kept])
        F[0, :] = 0.0
        f = GpuTableau(P, context=g.context)
        f.upload(F, vrow, vcol[kept])
        t1 = time.perf_counter()
        tg = targets_of(vrow, vcol, kept)
        out = f.scenario_batch([(1, lab, float(-s)) for lab, s in tg], list(range(len(tg) + 1)), check_cycles=True)
        t2 = time.perf_counter()
        f.close()
        return (t1 - t0) * 1e3, (t2 - t1) * 1e3, kept, tg, out

    device(), host()  # warm-up: kernel attributes, scratch buffers, the allocator
    dev, hst = [], []
    for _ in range(reps):
        dev.append(device())
        hst.append(host())
    _, _, kept, tg, out = dev[-1]
    same = all(np.array_equal(d[2], h[2]) and np.array_equal(d[4]["status"], h[4]["status"]) and
               np.array_equal(d[4]["rhs"].view(np.uint64), h[4]["rhs"].view(np.uint64)) for d, h in zip(dev, hst))

    pivots = out["p1"] + out["p2"]
    g.close()
    face_ms, batch_ms = [d[0] for d in dev], [d[1] for d in dev]
    hface_ms, hbatch_ms = [h[0] for h in hst], [h[1] for h in hst]
    total = [a + b_ for a, b_ in zip(face_ms, batch_ms)]
    htotal = [a + b_ for a, b_ in zip(hface_ms, hbatch_ms)]
    Wk = len(kept)
    return {"tableau": f"{H}x{W}", "face": f"{H}x{Wk}", "free": Wk - 1, "lps": len(tg), "solve_ms": solve_ms,
            "statuses": {str(s): int((out["status"] == s).sum()) for s in range(4)},
            "pivots_mean": float(pivots.mean()), "pivots_max": int(pivots.max()),
            "face_ms": spread(face_ms), "batch_ms": spread(batch_ms), "device_total_ms": spread(total),
            "host_face_ms": spread(hface_ms), "host_batch_ms": spread(hbatch_ms), "host_total_ms": spread(htotal),
            "face_bytes": 12 * W + 16 * (H - 1) * Wk + 4 * H, "download_bytes": 8 * H * W,
            "device_equals_host_bits": bool(same), "reps": reps,
            "not_measured": ["one fresh Solve() per target with an added objective = z* row"]}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="150x120,550x600,2000x2000", help="comma-separated VARSxCONS")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=12345)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only measures on the GPU")
    dev, cond = torch.cuda.get_device_name(0), gpu_conditions()
    for shape in a.sizes.split(","):
        nv, nc = (int(x) for x in shape.split("x"))
        out = run_size(nv, nc, a.reps, a.seed)
        out.update(device=dev, **cond)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

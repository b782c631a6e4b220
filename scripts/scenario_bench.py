"""Time what-if scenarios on one GPU: jslp_scenario_batch against the two ways a user answers the same question
without it.

For each size, solves a seeded dense packing LP (bench.py's generator) once and draws seeded scenarios: +-10 % on the
right-hand sides of up to three binding rows and on the costs of up to three basic variables.  Three arms, each timed
on the host clock around work that ends in a synchronise:
  batch       one GpuTableau.scenario_batch call (Solution.scenarios() without the name resolution and shaping)
  sequential  on the solved tableau: restore() the saved optimum, updateRightHandSide / updateCost, simplex(), per
              scenario (the reference's dynamic-modification path plus the undo)
  fresh       a fresh upload and simplex() of each edited initial tableau
Checks that batch and sequential agree bit for bit (status and final right-hand-side column) and that the fresh solves
reach the same verdict and objective to 1e-9 relative.  Prints one JSON line per size with the device name and power
limit beside the numbers.

    python scripts/scenario_bench.py [--sizes 150x120:300,550x600:24,2000x2000:4] [--seed 12345]
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


def scenarios_of(g, it, n, rng):
    import numpy as np
    g._cache.clear()
    M, vr, vc = g.matrix2d(), np.array(g.varIndexByRow), np.array(g.varIndexByCol)
    H, W = it.matrix.shape
    slack_row = {int(it.varIndexByRow[r]): r for r in range(1, H)}
    var_col = {int(it.varIndexByCol[c]): c for c in range(1, W)}
    binding = [int(v) for v in vc[1:] if int(v) in slack_row]
    basic = [int(v) for v in vr[1:] if int(v) in var_col]
    out = []
    for _ in range(n):
        sc = [(0, int(lab), float(it.matrix[slack_row[int(lab)], 0]) * rng.uniform(-0.1, 0.1))
              for lab in rng.choice(binding, size=min(3, len(binding)), replace=False)]
        sc += [(1, int(lab), float(it.matrix[0, var_col[int(lab)]]) * rng.uniform(-0.1, 0.1))
               for lab in rng.choice(basic, size=min(3, len(basic)), replace=False)]
        out.append(sc)
    return out, slack_row, var_col


def run_size(n_vars, n_cons, n_scen, seed):
    import numpy as np
    from jslpsolver_b200 import problems
    from jslpsolver_b200.tableau import GpuTableau
    it = problems.dense_packing_lp_tableau(n_vars, n_cons, seed)
    g = GpuTableau(1e-8)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol)
    g.simplex()
    assert g.feasible and g.bounded, "the benchmark LP has no optimum"
    H, W = g.height, g.width
    scen, slack_row, var_col = scenarios_of(g, it, n_scen, np.random.default_rng(seed))
    edits, offsets = [], [0]
    for sc in scen:
        edits += sc
        offsets.append(len(edits))
    g.scenario_batch(edits[:offsets[1]], offsets[:2])  # warm-up: kernel attributes, scratch buffers
    t0 = time.perf_counter()
    batch = g.scenario_batch(edits, offsets)
    batch_ms = (time.perf_counter() - t0) * 1e3

    g.save()
    seq_status, seq_rhs = [], []
    t0 = time.perf_counter()
    for sc in scen:
        g.restore()
        for kind, index, d in sc:
            (g.updateRightHandSide if kind == 0 else g.updateCost)(index, d)
        g.simplex()
        st = g.lastStatus
        seq_status.append(3 if st.cycled else 1 if not st.feasible else 2 if not st.bounded else 0)
        seq_rhs.append(g.rhs_column().copy())
    seq_ms = (time.perf_counter() - t0) * 1e3
    g.restore()

    fresh_ok, fresh_ms = True, 0.0
    for k, sc in enumerate(scen):
        Me = it.matrix.copy()
        for kind, index, d in sc:  # on the initial tableau every slack is basic and every variable non-basic
            if kind == 0:
                Me[slack_row[index], 0] -= d
            else:
                Me[0, var_col[index]] -= d
        t0 = time.perf_counter()
        f = GpuTableau(1e-8, context=g.context)
        f.upload(Me, it.varIndexByRow, it.varIndexByCol)
        f.simplex()
        raw = float(f.rhs_column()[0])
        fresh_ms += (time.perf_counter() - t0) * 1e3
        ok = bool(f.feasible and f.bounded) == (int(batch["status"][k]) == 0)
        if ok and f.feasible and f.bounded:
            want = float(batch["rhs"][k][0])
            ok = abs(raw - want) <= 1e-9 * max(1.0, abs(want))
        fresh_ok &= ok
        f.close()
    same = (list(batch["status"]) == seq_status and
            all(np.array_equal(batch["rhs"][k].view(np.uint64), seq_rhs[k].view(np.uint64)) for k in range(n_scen)))
    pivots = batch["p1"] + batch["p2"]
    g.close()
    return {"tableau": f"{H}x{W}", "scenarios": n_scen, "edits": len(edits),
            "statuses": {str(s): int((batch["status"] == s).sum()) for s in range(4)},
            "pivots_mean": float(pivots.mean()), "pivots_max": int(pivots.max()),
            "batch_ms": batch_ms, "sequential_ms": seq_ms, "fresh_ms": fresh_ms,
            "batch_us_per_scenario": 1e3 * batch_ms / n_scen,
            "speedup_vs_sequential": seq_ms / batch_ms, "speedup_vs_fresh": fresh_ms / batch_ms,
            "batch_equals_sequential_bits": bool(same), "fresh_agrees_1e-9": bool(fresh_ok)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="150x120:300,550x600:24,2000x2000:4",
                    help="comma-separated VARSxCONS:SCENARIOS")
    ap.add_argument("--seed", type=int, default=12345)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only measures on the GPU")
    dev, pw = torch.cuda.get_device_name(0), power_limit_w()
    for spec in a.sizes.split(","):
        shape, n = spec.split(":")
        nv, nc = (int(x) for x in shape.split("x"))
        out = run_size(nv, nc, int(n), a.seed)
        out.update(device=dev, power_limit_w=pw)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

"""Time parametric paths on bench.py's dense 2000x2000 LP (BASELINE.json configs[2]) on one GPU.

Solves the LP once, then for two paths:
  rhs   the binding row with the largest dual moves its right-hand side to 4x its value
  cost  the first basic structural variable moves its cost to 2x its value
times one jslp_parametric call after a warm-up call (CUDA events on the library's stream; the call ends in a
synchronise), and what a user does without it: a fresh upload and simplex() of the edited tableau at the end value
(host clock around work that ends in a synchronise).  Checks that both end results agree to 1e-9 relative.  Prints one
JSON line with the device name and power limit beside the numbers.  theta is in tableau units (the packing LP
maximises and has only `max` rows).  Algorithmic bytes per breakpoint: the pivot's 16 H W plus the selection's
56 H + 32 W (rhs) or 24 H + 64 W (cost).

    python scripts/parametric_bench.py [--n 2000] [--m 2000] [--cap 0 (= 4 (H + W))]
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


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2000, help="variables")
    ap.add_argument("--m", type=int, default=2000, help="constraints")
    ap.add_argument("--seed", type=int, default=12345)
    ap.add_argument("--cap", type=int, default=0, help="breakpoint cap (0 = 4 (H + W))")
    a = ap.parse_args()

    import numpy as np
    import torch
    from jslpsolver_b200 import problems
    from jslpsolver_b200.tableau import GpuTableau
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only measures on the GPU")

    it = problems.dense_packing_lp_tableau(a.n, a.m, a.seed)
    g = GpuTableau(1e-8)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol)
    g.simplex()
    st = g.lastStatus
    assert st.feasible and st.bounded, "the benchmark LP has no optimum"
    H, W = g.height, g.width
    cap = a.cap or 4 * (H + W)
    M, vr, vc = g.matrix2d(), np.array(g.varIndexByRow), np.array(g.varIndexByCol)
    slack_row = {int(it.varIndexByRow[r]): r for r in range(1, H)}
    var_col = {int(it.varIndexByCol[c]): c for c in range(1, W)}
    lab_r = max((abs(M[0, c]), int(vc[c])) for c in range(1, W) if int(vc[c]) in slack_row)[1]
    lab_c = next(int(vr[r]) for r in range(1, H) if int(vr[r]) in var_col)
    r0, c0 = slack_row[lab_r], var_col[lab_c]
    stream = torch.cuda.ExternalStream(g.context.lib.jslp_ctx_stream(g.context.handle))
    L = g.context.lib

    def fresh(edit):
        Me = it.matrix.copy()
        edit(Me)
        t0 = time.perf_counter()
        f = GpuTableau(1e-8, context=g.context)
        f.upload(Me, it.varIndexByRow, it.varIndexByCol)
        f.simplex()
        ms = (time.perf_counter() - t0) * 1e3
        raw = float(f.rhs_column()[0])
        f.close()
        return ms, raw

    out = {"workload": f"dense {a.n}x{a.m} seed {a.seed}, tableau {H}x{W}, solve {st.phase1_pivots + st.phase2_pivots} pivots",
           "device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "cap": cap}
    for kind, lab, theta0, target, edit in (
            ("rhs", lab_r, float(it.matrix[r0, 0]), 4.0 * float(it.matrix[r0, 0]), lambda Me: Me.__setitem__((r0, 0), 4.0 * it.matrix[r0, 0])),
            ("cost", lab_c, float(it.matrix[0, c0]), 2.0 * float(it.matrix[0, c0]), lambda Me: Me.__setitem__((0, c0), 2.0 * it.matrix[0, c0]))):
        k = 0 if kind == "rhs" else 1
        g.parametric_path(k, [lab], [1.0], theta0, target, cap)  # warm-up: graph capture, first launches
        launches0 = L.jslp_ctx_launches(g.context.handle)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        p = g.parametric_path(k, [lab], [1.0], theta0, target, cap)
        e1.record(stream)
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        launches = L.jslp_ctx_launches(g.context.handle) - launches0
        n = len(p["theta"])
        fresh_ms, fresh_raw = fresh(edit)
        end_raw = float(p["obj_raw"][-1])
        sel = 56 * H + 32 * W if kind == "rhs" else 24 * H + 64 * W
        out[kind] = {"breakpoints": n, "stop": int(p["stop"]), "call_ms": ms, "ms_per_breakpoint": ms / max(1, n),
                     "launches": int(launches), "launches_per_breakpoint": launches / max(1, n),
                     "algorithmic_bytes_per_breakpoint": 16 * H * W + sel,
                     "gbs": (16 * H * W + sel) * n / (ms * 1e6) if n else None,
                     "fresh_solve_ms": fresh_ms, "speedup": fresh_ms / ms,
                     "end_agrees_1e-9": abs(end_raw - fresh_raw) <= 1e-9 * max(1.0, abs(fresh_raw)) if p["stop"] == 1 else None}
    print(json.dumps(out))
    g.close()


if __name__ == "__main__":
    main()

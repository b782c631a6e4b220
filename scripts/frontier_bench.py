"""Time two-objective frontiers on dense_packing_multi_model(n, m, 2) (profit against attr1, both `max`) on one GPU.

For each size: solve the first objective, then
  call       one jslp_frontier call after a warm-up call (host clock around work that ends in a synchronise), its
             breakpoints, pivots and vertices (the vertex rule of frontier.py, DESIGN.md section 2g)
  price      k_price_objective's mean kernel time from torch.profiler over 50 calls, and its algorithmic bytes
             8 W per row with a non-zero coefficient + 4 H (vrow) + 8 nonzero rows (coefficients) + 16 W (R2, E out)
  weighted   what a user does without it: one fresh upload and simplex() of the weighted-sum tableau, row 0 =
             (1 - w) C1 + w C2, at the middle of each reported vertex's weight interval (the JSON model build is left
             out, which favours this alternative)
Prints one JSON line per size with the device name and power limit beside the numbers.  Sizes are tableau H x W.

    python scripts/frontier_bench.py [--sizes 121x151,601x551,2001x2001]
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


def attr1(n, m, seed):
    """attr1 of problems.dense_packing_multi_model(n, m, 2, seed), drawn as it draws it."""
    import numpy as np
    rng = np.random.default_rng(seed)
    rng.integers(1, 21, size=(m, n)); rng.integers(100, 501, size=m); rng.integers(1, 51, size=n)
    return rng.integers(1, 51, size=(1, n)).astype(np.float64)[0]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="121x151,601x551,2001x2001")
    ap.add_argument("--seed", type=int, default=12345)
    a = ap.parse_args()

    import numpy as np
    import torch
    from jslpsolver_b200 import frontier, problems
    from jslpsolver_b200.tableau import GpuTableau
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only measures on the GPU")
    dev, pl = torch.cuda.get_device_name(0), power_limit_w()
    for size in a.sizes.split(","):
        H, W = (int(x) for x in size.split("x"))
        m, n = H - 1, W - 1
        it = problems.dense_packing_lp_tableau(n, m, a.seed)
        c2 = np.zeros(n + m)
        c2[m:] = attr1(n, m, a.seed)  # variables take labels m .. m + n - 1
        g = GpuTableau(1e-8)
        g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol)
        g.simplex()
        assert g.feasible and g.bounded
        cap = 4 * (H + W)
        g.frontier_path(c2, cap)  # warm-up: graph capture, first launches
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = g.frontier_path(c2, cap)
        call_ms = (time.perf_counter() - t0) * 1e3
        theta = [float(x) for x in out["theta"]]
        pts, starts = [], []
        for rhs, vrow, at in zip(out["pt_rhs"], out["pt_vrow"], out["pt_break"]):
            x = np.zeros(n)
            for r in range(1, H):
                if vrow[r] >= m:
                    x[vrow[r] - m] = rhs[r]
            pts.append(tuple(x))
            starts.append(0.0 if at == 0 else theta[at - 1])
        stop = frontier.STOPS[int(out["stop"])]
        verts = frontier.vertices(pts, starts, theta[-1], stop, 1e-8)
        pivots = int(sum(1 for r in out["rc_lbl"] if r[0] >= 0 and r[1] >= 0))

        M, vr = g.matrix2d(), np.array(g.varIndexByRow)
        nz = int(sum(1 for r in range(1, H) if c2[vr[r]] != 0))
        price_bytes = 8 * W * nz + 4 * H + 8 * nz + 16 * W
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(50):
                g.frontier_path(c2, 1)
            torch.cuda.synchronize()
        ks = [e for e in prof.events() if "k_price_objective" in e.name]
        price_us = sum(e.device_time for e in ks) / max(1, len(ks))

        c1 = it.matrix[0].copy()
        row2 = np.zeros(W)
        row2[1:] = c2[np.array(it.varIndexByCol[1:])]
        weighted_ms, agree = 0.0, True
        for pt, lo, hi in verts:
            w = (lo + hi) / 2
            Me = it.matrix.copy()
            Me[0] = (1 - w) * c1 + w * row2
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f = GpuTableau(1e-8, context=g.context)
            f.upload(Me, it.varIndexByRow, it.varIndexByCol)
            f.simplex()
            raw = float(f.rhs_column()[0])
            weighted_ms += (time.perf_counter() - t0) * 1e3
            f.close()
            x = np.array(pt)
            want = (1 - w) * float(attr_row(it, m) @ x) + w * float(c2[m:] @ x)
            agree &= abs(-raw - want) <= 1e-9 * max(1.0, abs(want))  # row 0 holds minus the maximised value
        print(json.dumps({"size": f"{H}x{W}", "device": dev, "power_limit_w": pl, "solve_pivots":
                          g.lastStatus.phase1_pivots + g.lastStatus.phase2_pivots, "breakpoints": len(theta),
                          "pivots": pivots, "points": int(out["n_points"]), "vertices": len(verts), "stop": stop,
                          "call_ms": call_ms, "ms_per_pivot": call_ms / max(1, pivots),
                          "price_us": price_us, "price_launches": len(ks), "price_rows": nz, "price_bytes": price_bytes,
                          "price_gbs": price_bytes / (price_us * 1e3) if price_us else None,
                          "weighted_solves_ms": weighted_ms, "weighted_solves": len(verts),
                          "weighted_agree_1e-9": bool(agree)}))
        g.close()


def attr_row(it, m):
    """The first objective (profit) by variable, from the tableau's row 0 (maximisation: +c)."""
    import numpy as np
    c = np.zeros(it.matrix.shape[1] - 1)
    for col in range(1, it.matrix.shape[1]):
        c[int(it.varIndexByCol[col]) - m] = it.matrix[0, col]
    return c


if __name__ == "__main__":
    main()

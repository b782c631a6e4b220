"""Time Solution.iis() on planted infeasible LPs (problems.planted_infeasible_model) on one GPU.

Two sizes: one whose rows fit the shared-memory batch (k_node_batch, one CTA per tested set) and one that does not
(tests run one after another on the HBM path).  Per size, two arms, alternated round by round after a warm-up:
  batched  Solution.iis() as shipped: speculative rounds one wave of co-resident CTAs wide, with the pre-pass
  literal  the one-row-at-a-time deletion filter (width 1, no pre-pass)
Both arms must return the same rows.  Also times one jslp_feasibility_batch call testing every one-row-smaller
subset of all rows (the raw batch throughput; at the HBM size only the first --hbm-sets of them).  Prints one JSON line
with the device name and power limit beside the numbers.

    python scripts/iis_bench.py [--rounds 3] [--k 6] [--seed 21]
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
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--k", type=int, default=6, help="rows in the planted conflict")
    ap.add_argument("--seed", type=int, default=21)
    ap.add_argument("--hbm-sets", type=int, default=20)
    a = ap.parse_args()

    import numpy as np
    import torch
    from jslpsolver_b200 import Solve, problems
    from jslpsolver_b200.iis import compute
    from jslpsolver_b200.tableau import GpuTableau
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only measures on the GPU")

    out = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "sizes": {}}
    for label, n, m in (("k2", 150, 120), ("hbm", 550, 600)):
        jm = problems.planted_infeasible_model(n, m, a.k, a.seed)
        sol = Solve(jm, full=True)
        assert not sol.feasible
        arms = {"batched": lambda: compute(sol), "literal": lambda: compute(sol, width=1, prepass=False)}
        res = {name: f() for name, f in arms.items()}  # warm-up
        times = {name: [] for name in arms}
        for _ in range(a.rounds):
            for name, f in arms.items():
                t0 = time.perf_counter()
                r = f()
                times[name].append((time.perf_counter() - t0) * 1e3)
                assert r == res[name]
        assert res["batched"]["constraints"] == res["literal"]["constraints"], "the two schedules disagree"
        row = {"tableau": f"{m + 1}x{n + 1}", "iis_rows": len(res["batched"]["constraints"])}
        for name in arms:
            best = min(times[name])
            row[name] = {"ms_min": best, "ms_max": max(times[name]), "lps": res[name]["lps"],
                         "lps_per_s": res[name]["lps"] / best * 1e3}

        # raw batch: every one-row-smaller subset of all rows in one call
        it = sol._tableau.model.initial_tableau()
        H = it.matrix.shape[0]
        g = GpuTableau(sol._tableau.model.precision)
        g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted)
        g.save()
        n_sets = H - 1 if label == "k2" else min(H - 1, a.hbm_sets)
        keep = np.ones((n_sets, H), dtype=np.uint8)
        keep[np.arange(n_sets), 1 + np.arange(n_sets)] = 0
        g.feasibility_batch(keep)  # warm-up
        ts = []
        for _ in range(a.rounds):
            t0 = time.perf_counter()
            v, p = g.feasibility_batch(keep)
            ts.append((time.perf_counter() - t0) * 1e3)
        g.close()
        row["batch_minus_one"] = {"sets": n_sets, "ms_min": min(ts), "ms_max": max(ts),
                                  "lps_per_s": n_sets / min(ts) * 1e3, "mean_phase1_pivots": float(np.mean(p))}
        out["sizes"][label] = row
    print(json.dumps(out))


if __name__ == "__main__":
    main()

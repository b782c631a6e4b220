"""Solution.unbounded() on the device for problems.planted_unbounded_model at two sizes: 150 x 120 with 8 leak
variables (4 solo leaks, 2 pairs; the cone LPs run one CTA each in shared memory) and 2001 x 2001 with the same leaks
(the cone LPs run one after another on the single-tableau path).  Per size and run:

  solve      the cold Solve(model, full=True) that ends unbounded
  report     the ray and row report (one column and column 0 of the stop tableau)
  cone       jslp_cone_create
  additive   the additive phase: LPs, pivots, time
  deletion   the deletion filter: waves (launches of jslp_column_batch), LPs, pivots, time
  total      Solution.unbounded() end to end, as a user calls it

GPU name, power limit and clocks are read in the same run.  Usage: python scripts/unbounded_bench.py [--runs 2]
[--sizes small,large]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = {"small": (120, 150, 4, 2), "large": (2000, 2000, 4, 2)}  # (variables, rows, solo leaks, pairs)


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


def run(jm) -> dict:
    import jslpsolver_b200 as J
    from jslpsolver_b200 import iis, unbounded as U
    from jslpsolver_b200.tableau import GpuTableau
    sol, t_solve = timed(lambda: J.Solve(jm, full=True))
    assert not sol.bounded, "the planted model did not end unbounded"
    t = sol._tableau
    m = t.model
    P = m.precision
    it = m.initial_tableau()
    H, W = it.matrix.shape
    _, t_report = timed(lambda: U.ray_report(m, it, t.rhs_column(), t.varIndexByRow, t.varIndexByCol,
                                             t.unboundedVarIndex, t.column(int(np.nonzero(
                                                 t.varIndexByCol == t.unboundedVarIndex)[0][0])), P))
    structural = {v.index for v in m.variables}
    col_of_label = {int(it.varIndexByCol[c]): c for c in range(1, W) if int(it.varIndexByCol[c]) in structural}
    scratch = GpuTableau(P, context=t.context)
    scratch.upload(it.matrix, it.varIndexByRow, it.varIndexByCol, it.unrestricted)
    cone, t_cone = timed(scratch.cone)
    cone.save()
    phase = {"name": "additive"}
    stats = {k: {"lps": 0, "pivots": 0, "waves": 0, "ms": 0.0} for k in ("additive", "deletion")}

    def test_batch(sets):
        keep = np.ones((len(sets), W), dtype=np.uint8)
        for i, s in enumerate(sets):
            keep[i, list(s)] = 0
        keep[:, 0] = 1
        res, ms = timed(lambda: cone.column_batch(keep))
        st = stats[phase["name"]]
        st["lps"] += len(sets)
        st["pivots"] += int(res["pivots"].sum())
        st["waves"] += 1
        st["ms"] += ms
        out = [(U.verdict(int(res["status"][i]), float(res["eval_raw"][i]), P),
                U.support(res["rhs"][i], res["vrow"][i], col_of_label, P)) for i in range(len(sets))]
        if phase["name"] == "additive" and out[0][0] == U.BOUNDED:
            phase["name"] = "deletion"  # the additive phase ends at its first bounded test
        return out

    K = iis.wave_width(cone.context, H + 1, W)
    (confirmed, cols, irreducible), _ = timed(lambda: U.bounding_set(test_batch, len(col_of_label), K))
    cone.close()
    scratch.close()
    total, t_total = timed(lambda: sol.unbounded())
    return {"tableau": [H, W], "solve_ms": round(t_solve, 2), "report_ms": round(t_report, 3),
            "cone_ms": round(t_cone, 3), "wave_width": K,
            "additive": {k: round(v, 2) if isinstance(v, float) else v for k, v in stats["additive"].items()},
            "deletion": {k: round(v, 2) if isinstance(v, float) else v for k, v in stats["deletion"].items()},
            "total_ms": round(t_total, 2), "lps": total["lps"], "confirmed": confirmed,
            "bound": None if cols is None else len(cols), "irreducible": irreducible}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--sizes", default="small,large")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    a = ap.parse_args()
    from jslpsolver_b200 import problems
    lines = [{"gpu": gpu_info()}]
    print(json.dumps(lines[0]), flush=True)
    for name in a.sizes.split(","):
        n_vars, n_cons, n_solo, n_pairs = SIZES[name]
        jm = problems.planted_unbounded_model(n_vars, n_cons, n_solo, n_pairs, seed=1)
        for r in range(a.runs):
            rec = dict(size=name, run=r, **run(jm))
            lines.append(rec)
            print(json.dumps(rec), flush=True)
    lines.append({"gpu": gpu_info()})
    print(json.dumps(lines[-1]), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()

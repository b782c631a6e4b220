"""Time the sensitivity bounds of bench.py's dense 2000x2000 LP (BASELINE.json configs[2]) on one GPU.

Solves the LP once, then times over many calls after a warm-up:
  call      jslp_sensitivity (key reset, one pass over the tableau, the bounds read back, synchronise), with CUDA
            events on the library's stream
  download  what a user can do without it: jslp_download of the whole tableau plus oracle/sensitivity.py's NumPy
            restatement of the same bounds (host clock; the download ends in a synchronise), and the download alone
and checks that both give the same bits.  Prints one JSON line with the device name and power limit beside the
numbers; the algorithmic bytes of the device pass are 8 (H-1) W + 8 (H+W) + 32 (H+W).

    python scripts/sensitivity_bench.py [--n 2000] [--m 2000] [--iters 200] [--warmup 20]
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
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--download-iters", type=int, default=10)
    a = ap.parse_args()

    import numpy as np
    import torch
    from jslpsolver_b200 import problems
    from jslpsolver_b200.tableau import GpuTableau
    from oracle import sensitivity as S
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only measures on the GPU")

    it = problems.dense_packing_lp_tableau(a.n, a.m, a.seed)
    g = GpuTableau(1e-8)
    g.upload(it.matrix, it.varIndexByRow, it.varIndexByCol)
    g.simplex()
    st = g.lastStatus
    assert st.feasible and st.bounded, "the benchmark LP has no optimum"
    H, W = g.height, g.width
    L, h = g.context.lib, g.handle
    stream = torch.cuda.ExternalStream(L.jslp_ctx_stream(g.context.handle))
    cl, ch, rl, rh = (np.empty(W), np.empty(W), np.empty(H), np.empty(H))
    call = lambda: L.jslp_sensitivity(h, cl.ctypes.data, ch.ctypes.data, rl.ctypes.data, rh.ctypes.data)

    for _ in range(a.warmup):
        assert call() == 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(a.iters):
        assert call() == 0
    e1.record(stream)
    e1.synchronize()
    device_ms = e0.elapsed_time(e1) / a.iters

    def download_path():
        g._cache.clear()
        M = g.matrix2d()
        return S.bounds(M, g.varIndexByRow, g.varIndexByCol, None, g.precision)

    want = download_path()
    t0 = time.perf_counter()
    for _ in range(a.download_iters):
        want = download_path()
    download_ms = (time.perf_counter() - t0) * 1e3 / a.download_iters
    g._cache.clear()
    M = g.matrix2d()
    t0 = time.perf_counter()
    for _ in range(a.download_iters):
        g._cache.clear()
        g.matrix2d()
    copy_ms = (time.perf_counter() - t0) * 1e3 / a.download_iters
    same = all(np.array_equal(x.view(np.uint64), y.view(np.uint64)) for x, y in zip((cl, ch, rl, rh), want))

    algo_bytes = 8 * (H - 1) * W + 8 * (H + W) + 32 * (H + W)
    print(json.dumps({
        "workload": f"dense {a.n}x{a.m} seed {a.seed}, tableau {H}x{W}, {st.phase1_pivots + st.phase2_pivots} pivots",
        "device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
        "sensitivity_call_ms": device_ms, "call_gbs": algo_bytes / device_ms / 1e6, "algorithmic_bytes": algo_bytes,
        "download_plus_numpy_ms": download_ms, "download_only_ms": copy_ms, "speedup": download_ms / device_ms,
        "bit_identical": bool(same), "matrix_bytes": int(M.nbytes)}))
    g.close()


if __name__ == "__main__":
    main()

"""Builds libjslp_b200.so (sm_90a, H100) in-tree with nvcc.  No GPU is needed to compile."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "jslp_api.cu")
DEPS = [SRC] + [os.path.join(HERE, "csrc", f) for f in ("jslp_kernels.cuh", "jslp_step.cuh", "jslp_node_kernel.cuh", "jslp_slots.cuh", "jslp_dynamic.cuh", "jslp_comm.cuh", "jslp_bnb_enhanced.cuh", "jslp_batch.cuh", "jslp_bnb.cuh", "jslp_sensitivity.cuh", "jslp_iis.cuh", "jslp_parametric.cuh", "jslp_scenario.cuh", "jslp_recourse.cuh", "jslp_crash.cuh", "jslp_frontier.cuh", "jslp_face.cuh", "jslp_bound.cuh", "jslp_lex.cuh", "jslp_elastic.cuh", "jslp_cone.cuh", "jslp_pool.cuh", "jslp_conflict.cuh", "jslp_forest.cuh", "jslp_frontier.h", "jslp_cycles.h", "jslp_hostmath.h")] + [
    os.path.join(os.path.dirname(HERE), "include", "jslp_b200.h")]
OUT = os.path.join(HERE, "libjslp_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-fmad=false",                 # JS has no FMA: never contract a*b-c (SURVEY.md 3.6)
    "-Xcompiler", "-fPIC", "-shared", "-cudart", "shared",
]


def nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libjslp_b200.so cannot be built (there is no CPU fallback)")


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in DEPS):
        return OUT
    cmd = [nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT, SRC]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building libjslp_b200.so")
    if verbose:
        sys.stderr.write(res.stdout + res.stderr)
    return OUT


if __name__ == "__main__":
    print(build(force=True, verbose="-v" in sys.argv))

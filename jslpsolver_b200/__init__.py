"""jslpsolver_b200 -- H100-native (sm_90a) dense-tableau simplex + branch-and-cut behind
jsLPSolver's `solver.Solve()` JSON-model API.  The numerical path is hand-written CUDA in
libjslp_b200.so (C ABI: include/jslp_b200.h); there is no CPU fallback."""
from ._lib import JslpError, load as load_library  # noqa: F401
from .model import Model  # noqa: F401
from .solver import Conflict, Frontier, FrontierMIP, Lexicographic, LexicographicMIP, Pool, Repair, RepairMIP, Scenarios, Solve, Solver, TwoStage, Variability, solver  # noqa: F401
from .tableau import DeviceContext, GpuTableau, default_context  # noqa: F401

__all__ = ["Solve", "Conflict", "Frontier", "FrontierMIP", "Lexicographic", "LexicographicMIP", "Pool", "Repair", "RepairMIP", "Scenarios", "TwoStage", "Variability", "Solver", "solver", "Model", "GpuTableau", "DeviceContext",
           "default_context", "JslpError", "load_library"]

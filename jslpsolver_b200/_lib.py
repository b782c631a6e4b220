"""ctypes binding of libjslp_b200.so (include/jslp_b200.h).  Fails loudly when the CUDA
extension is missing or no GPU is present: there is no CPU fallback in this package."""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

_LIB = None

OPT_ENGINE, OPT_BATCH, OPT_PIVOT_LOG_CAP = 1, 2, 3
OPT_STEP_VARIANT, OPT_GRID_PER_SM, OPT_LOOKAHEAD, OPT_TIMELINE, OPT_PDL, OPT_PINGPONG = 4, 5, 6, 7, 8, 9
OPT_NODE_SLOTS, OPT_SLOT_STEPS, OPT_SLOT_VARIANT, OPT_USE_MIR_CUTS, OPT_NODE_LOG_CAP = 10, 11, 12, 13, 14
ENGINE_AUTO, ENGINE_TWO_KERNEL, ENGINE_FUSED, ENGINE_PERSISTENT, ENGINE_RESIDENT = 0, 1, 2, 3, 4


class JslpError(RuntimeError):
    pass


class LpStatus(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "feasible", "bounded", "cycled", "cycle_start", "cycle_length", "phase1_pivots",
        "phase2_pivots", "unbounded_var_index", "simplex_iters", "width", "height", "engine")] + [
        ("evaluation_raw", C.c_double), ("evaluation", C.c_double), ("best_possible_eval", C.c_double),
        ("gpu_ms", C.c_double), ("kernel_launches", C.c_int64)]


class Cut(C.Structure):
    _fields_ = [("type", C.c_int32), ("var_index", C.c_int32), ("value", C.c_double)]


class ScenarioEdit(C.Structure):  # jslp_scenario_edit
    _fields_ = [("kind", C.c_int32), ("index", C.c_int32), ("difference", C.c_double)]


class Fix(C.Structure):  # jslp_fix
    _fields_ = [("column", C.c_int32), ("value", C.c_double)]


ALL_GATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int64)


class BnbOpts(C.Structure):
    _fields_ = [("tolerance", C.c_double), ("is_minimization", C.c_int32), ("check_cycles", C.c_int32),
                ("max_spec_batch", C.c_int32), ("rank", C.c_int32), ("n_ranks", C.c_int32),
                ("max_nodes", C.c_int64), ("all_gather", ALL_GATHER_FN), ("user", C.c_void_p),
                ("comm", C.c_void_p), ("shard_policy", C.c_int32), ("keep_solutions", C.c_int32),
                ("timeout_ms", C.c_double), ("service", C.c_int32), ("node_selection", C.c_int32),
                ("branching", C.c_int32), ("strong_candidates", C.c_int32)]


class BnbStatus(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("feasible", "bounded", "is_integral", "iterations", "n_best_cuts",
                                         "rounds")] + [
        ("nodes_evaluated", C.c_int64), ("pivots", C.c_int64), ("evaluation", C.c_double),
        ("best_possible_eval", C.c_double), ("gpu_ms", C.c_double), ("kernel_launches", C.c_int64),
        ("host_eval_ms", C.c_double), ("host_commit_ms", C.c_double),
        ("host_root_ms", C.c_double), ("host_final_ms", C.c_double), ("node_kernel_ms", C.c_double),
        ("timed_out", C.c_int32), ("n_solutions", C.c_int32), ("nodes_pruned", C.c_int64),
        ("collectives", C.c_int64), ("slot_pivots", C.c_int64), ("slot_ms", C.c_double), ("slot_bytes", C.c_double),
        ("cycle_redos_kernel", C.c_int64), ("cycle_redos_slots", C.c_int64), ("cycle_redos_pruned", C.c_int64)]


class StartStatus(C.Structure):  # jslp_start_status
    _fields_ = [("status", C.c_int32), ("n_cuts", C.c_int32), ("nodes", C.c_int64), ("pivots", C.c_int64),
                ("evaluation", C.c_double)]


START_SEED, START_FEASIBLE, START_INFEASIBLE, START_INCOMPLETE, START_SKIPPED = 0, 1, 2, 3, 4


# every symbol include/jslp_b200.h declares: (name, restype, argtypes)
P = C.c_void_p
SYMBOLS = [
    ("jslp_last_error", C.c_char_p, []),
    ("jslp_abi_version", C.c_int, []),
    ("jslp_ctx_create", C.c_int, [C.c_int, P, C.POINTER(P)]),
    ("jslp_ctx_destroy", None, [P]),
    ("jslp_ctx_stream", P, [P]),
    ("jslp_ctx_launches", C.c_int64, [P]),
    ("jslp_ctx_sync", C.c_int, [P]),
    ("jslp_tab_create", C.c_int, [P, C.c_int, C.c_int, C.c_int, C.c_double, C.POINTER(P)]),
    ("jslp_tab_destroy", None, [P]),
    ("jslp_tab_upload", C.c_int, [P, P, P, P, P, C.c_int, P, C.c_int, C.c_int, P]),
    ("jslp_tab_set_option", C.c_int, [P, C.c_int, C.c_double]),
    ("jslp_debug_timeline", C.c_int, [P, P, C.c_int64, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    ("jslp_debug_copy_gbs", C.c_int, [P, C.c_int64, C.c_int, C.POINTER(C.c_double)]),
    ("jslp_simplex", C.c_int, [P, C.c_int, C.POINTER(LpStatus)]),
    ("jslp_phase1", C.c_int, [P, C.c_int, C.POINTER(LpStatus)]),
    ("jslp_phase2", C.c_int, [P, C.c_int, C.POINTER(LpStatus)]),
    ("jslp_pivot", C.c_int, [P, C.c_int, C.c_int]),
    ("jslp_save", C.c_int, [P]),
    ("jslp_restore", C.c_int, [P]),
    ("jslp_add_cuts", C.c_int, [P, P, C.c_int]),
    ("jslp_apply_cuts", C.c_int, [P, P, C.c_int, C.c_int, C.POINTER(LpStatus)]),
    ("jslp_add_mir_cut", C.c_int, [P, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    ("jslp_apply_mir_cuts", C.c_int, [P, C.POINTER(C.c_int)]),
    ("jslp_fractional_volume", C.c_int, [P, C.c_int, C.POINTER(C.c_double)]),
    ("jslp_put_in_base", C.c_int, [P, C.c_int, C.POINTER(C.c_int)]),
    ("jslp_take_out_of_base", C.c_int, [P, C.c_int, C.POINTER(C.c_int)]),
    ("jslp_update_rhs", C.c_int, [P, C.c_int, C.c_double]),
    ("jslp_update_coefficient", C.c_int, [P, C.c_int, C.c_int, C.c_double]),
    ("jslp_update_cost", C.c_int, [P, C.c_int, C.c_int, C.c_double]),
    ("jslp_add_constraint", C.c_int, [P, C.c_int, C.c_double, C.c_int, P, P, C.c_int]),
    ("jslp_remove_constraint", C.c_int, [P, C.c_int]),
    ("jslp_add_variable", C.c_int, [P, C.c_int, C.c_double, C.c_int, C.c_int, C.c_int]),
    ("jslp_tab_info", C.c_int, [P, P]),
    ("jslp_remove_variable", C.c_int, [P, C.c_int]),
    ("jslp_is_integral", C.c_int, [P, C.POINTER(C.c_int)]),
    ("jslp_most_fractional", C.c_int, [P, C.POINTER(C.c_int32), C.POINTER(C.c_double)]),
    ("jslp_download", C.c_int, [P, P, P, P, P, P, P, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    ("jslp_pivot_log", C.c_int, [P, P, C.c_int, C.POINTER(C.c_int)]),
    ("jslp_sensitivity", C.c_int, [P, P, P, P, P]),
    ("jslp_feasibility_batch", C.c_int, [P, P, C.c_int, P, P]),
    ("jslp_parametric", C.c_int, [P, C.c_int, P, P, C.c_int, C.c_double, C.c_double, C.c_int, P, P, P, P,
                                  C.POINTER(C.c_int), C.POINTER(C.c_int), P, P]),
    ("jslp_scenario_batch", C.c_int, [P, P, P, C.c_int, C.c_int, P, P, P, P, P, P]),
    ("jslp_recourse_batch", C.c_int, [P, P, P, C.c_int, P, C.c_int, P, C.c_int, C.c_int, P, P, P, P, P, P, P, P]),
    ("jslp_crash", C.c_int, [P, P, C.c_int, P, P, C.POINTER(C.c_int)]),
    ("jslp_frontier", C.c_int, [P, P, C.c_int, C.c_int, P, P, P, P, P, P, C.POINTER(C.c_int), C.POINTER(C.c_int), P, P,
                                P, C.POINTER(C.c_int), P, P]),
    ("jslp_face_create", C.c_int, [P, C.POINTER(P), C.POINTER(C.c_int32), P]),
    ("jslp_bound_create", C.c_int, [P, C.c_double, C.POINTER(P)]),
    ("jslp_lex_next", C.c_int, [P, P, C.c_double, C.POINTER(P), C.POINTER(C.c_int32), P]),
    ("jslp_elastic_create", C.c_int, [P, P, P, C.c_int, C.POINTER(P), C.POINTER(C.c_int32)]),
    ("jslp_cone_create", C.c_int, [P, C.POINTER(P)]),
    ("jslp_column_batch", C.c_int, [P, P, C.c_int, P, P, P, P, P]),
    ("jslp_column", C.c_int, [P, C.c_int, P]),
    ("jslp_pool_batch", C.c_int, [P, P, P, P, P, C.c_int, C.c_int, C.c_int, P, P, P, P, P, P, P, P]),
    ("jslp_target_batch", C.c_int, [P, P, P, P, P, C.c_int, C.c_int, C.c_int, P, P, P, P, P, P, P, P]),
    ("jslp_box_batch", C.c_int, [P, P, P, P, P, C.c_int, C.c_int, C.c_int, P, P, P, P, P, P, P, P]),
    ("jslp_conflict_batch", C.c_int, [P, P, P, P, P, C.c_int, C.c_int, P, P, P, P, P, P, P]),
    ("jslp_branch_and_cut", C.c_int, [P, C.POINTER(BnbOpts), C.POINTER(BnbStatus), P, C.c_int]),
    ("jslp_branch_and_cut_start", C.c_int, [P, C.POINTER(BnbOpts), P, P, C.c_int, C.c_int64, P,
                                            C.POINTER(BnbStatus), P, C.c_int]),
    ("jslp_bnb_batch", C.c_int, [P, P, P, C.c_int, C.POINTER(BnbOpts), C.c_int, P, P, P, P]),
    ("jslp_bnb_node_log", C.c_int, [P, P, C.c_int64, C.POINTER(C.c_int64)]),
    ("jslp_bnb_solution", C.c_int, [P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int32), P, P, C.c_int]),
    ("jslp_comm_unique_id", C.c_int, [P]),
    ("jslp_comm_create", C.c_int, [P, P, C.c_int, C.c_int, C.POINTER(P)]),
    ("jslp_comm_destroy", None, [P]),
    ("jslp_comm_all_gather", C.c_int, [P, P, C.c_int64]),
    ("jslp_comm_all_reduce_min", C.c_int, [P, P, C.c_int]),
]


def lib_path() -> str:
    return _build.OUT


def load(build_if_missing: bool = True):
    """Loads the shared library (building it with nvcc when stale/missing).  Raises if absent."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if build_if_missing:
        try:
            path = _build.build()
        except Exception as e:  # stale-but-present library on a box without nvcc is still usable
            if not os.path.exists(path):
                raise JslpError(f"libjslp_b200.so is missing and could not be built: {e}") from e
    if os.environ.get("JSLP_LIB"):  # A/B builds of the same ABI (tuning aid)
        path = os.environ["JSLP_LIB"]
    if not os.path.exists(path):
        raise JslpError("libjslp_b200.so is missing: run `python -m jslpsolver_b200.build` (no CPU fallback)")
    L = C.CDLL(path)
    for name, res, args in SYMBOLS:
        if os.environ.get("JSLP_LIB") and not hasattr(L, name):
            continue  # A/B against an older build of the library: newer entry points are simply absent
        fn = getattr(L, name)  # AttributeError here == ABI drift
        fn.restype = res
        fn.argtypes = args
    _LIB = L
    return L


def check(rc: int):
    if rc != 0:
        msg = load().jslp_last_error().decode(errors="replace")
        raise JslpError(f"libjslp_b200 error {rc}: {msg}")

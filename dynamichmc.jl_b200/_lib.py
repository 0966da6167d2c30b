"""ctypes binding of libdhmc_b200.so (include/dhmc.h) — the same entry points the
Julia shim binds with ccall (INTEGRATION.md).  No torch types cross this layer."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DHMC_B200_LIB", os.path.join(_HERE, "csrc", "libdhmc_b200.so"))

DHMC_OK, DHMC_EARG, DHMC_ENUMERIC, DHMC_ECUDA, DHMC_ENOMEM, DHMC_ENCCL = 0, 1, 2, 3, 4, 5
DHMC_CHAIN_BAD_INITIAL, DHMC_CHAIN_NONFINITE_Q, DHMC_CHAIN_LEAPFROG_NONFINITE = 1, 4, 64   # per-chain status bits (include/dhmc.h)
COMM_ID_BYTES = 128
FAMILY_STD_NORMAL, FAMILY_DIAG_NORMAL, FAMILY_FUNNEL, FAMILY_LOGISTIC, FAMILY_USER = 0, 1, 2, 3, 4
METRIC_NOTHING, METRIC_DIAGONAL, METRIC_SYMMETRIC, METRIC_SYMMETRIC_POOLED = 0, 1, 2, 3

tree_stats_dtype = np.dtype(
    [("pi", "<f8"), ("depth", "<i8"), ("left", "<i8"), ("right", "<i8"),
     ("acceptance_rate", "<f8"), ("steps", "<i8"), ("directions", "<u4"), ("pad", "<u4")])

EXPORTS = [
    "dhmc_create", "dhmc_destroy", "dhmc_last_error", "dhmc_get_layout", "dhmc_set_problem", "dhmc_set_problems", "dhmc_set_problems_ragged",
    "dhmc_user_family_name",
    "dhmc_family_available",
    "dhmc_set_position", "dhmc_random_position", "dhmc_set_metric", "dhmc_set_metric_dense",
    "dhmc_get_metric_dense", "dhmc_metric_is_dense", "dhmc_set_stepsize",
    "dhmc_set_momentum", "dhmc_get_state", "dhmc_chain_status", "dhmc_get_transition_count",
    "dhmc_set_transition_count", "dhmc_leapfrog", "dhmc_phase_logdensity", "dhmc_sample_tree",
    "dhmc_find_initial_stepsize", "dhmc_warmup_stage", "dhmc_mcmc", "dhmc_mcmc_from", "dhmc_mcmc_dev",
    "dhmc_tree_summary_dev", "dhmc_last_total_steps", "dhmc_last_kernel_ms", "dhmc_kernel_launches",
    "dhmc_ess_rhat_dev", "dhmc_ess_rhat_problems_dev", "dhmc_acceptance_quantiles_dev", "dhmc_mcmc_thinned", "dhmc_host_alloc", "dhmc_host_free",
    "dhmc_comm_unique_id", "dhmc_comm_init", "dhmc_comm_destroy", "dhmc_allgather_dev",
    "dhmc_allgather_positions_dev", "dhmc_last_comm_ms",
    "dhmc_mcmc_summary", "dhmc_summary_merge", "dhmc_summary_finish", "dhmc_mcmc_summary_histogram",
    "dhmc_histogram_quantiles",
]
# streaming summary record (include/dhmc.h DHMC_SUMMARY_*): numpy [P, D, SUMMARY_FIELDS] = column-major [F, D, P]
(SUMMARY_CHAINS, SUMMARY_NKEEP, SUMMARY_MEAN, SUMMARY_SS_SEQ, SUMMARY_M2, SUMMARY_SS_CHAIN, SUMMARY_BELOW,
 SUMMARY_FIELDS) = range(8)


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("family", C.c_int32), ("dim", C.c_int64),
                ("n_chains", C.c_int64), ("chain_offset", C.c_int64), ("seed", C.c_uint64),
                ("max_depth", C.c_int32), ("threads_per_chain", C.c_int32),
                ("min_delta", C.c_double), ("ctas_per_sm", C.c_int32), ("reserved", C.c_int32)]


class DualAveragingC(C.Structure):
    _fields_ = [("delta", C.c_double), ("gamma", C.c_double), ("kappa", C.c_double),
                ("t0", C.c_int32), ("pad", C.c_int32)]


class MissingExtension(ImportError):
    pass


_libs = {}


def lib(path=None):
    """Load libdhmc_b200.so (or, with `path`, a user-model build of it: compile_user_model in api.py).  Fails loudly when
    the CUDA extension is missing: there is no CPU fallback."""
    path = os.path.abspath(path or LIB_PATH)
    so = _libs.get(path)
    if so is None:
        if not os.path.exists(path):
            raise MissingExtension(
                f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (nvcc, sm_90a).  dynamichmc.jl_b200 has no CPU fallback.")
        so = C.CDLL(path)
        so.dhmc_last_error.restype = C.c_char_p
        so.dhmc_last_error.argtypes = [C.c_void_p]
        so.dhmc_mcmc_summary.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        so.dhmc_summary_merge.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64]
        so.dhmc_summary_finish.argtypes = [C.c_void_p, C.c_int64, C.c_int64] + [C.c_void_p] * 7
        so.dhmc_mcmc_summary_histogram.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        so.dhmc_histogram_quantiles.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_int64,
                                                C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        _libs[path] = so
    return so


def ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)

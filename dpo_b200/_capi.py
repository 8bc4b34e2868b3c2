"""ctypes binding of the C ABI in include/dpgo_b200.h (libdpgo_b200.so).

Fails loudly: if the shared library is missing or a CUDA device is not usable, every entry point
raises -- there is no CPU fallback in the product path.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libdpgo_b200.so")

OK = 0
STATUS_DOUBLES = 5            # DPGO_STATUS_DOUBLES: quad, lin, |rgrad|^2, relative change, optimising calls
ALG_RTR, ALG_RGD = 0, 1
PRECOND_NONE, PRECOND_BLOCK_JACOBI, PRECOND_DENSE_EXACT, PRECOND_SPARSE_EXACT = 0, 1, 2, 3
TCG_NAMES = {0: "NEGCURVTURE", 1: "EXCREGION", 2: "LCON", 3: "SCON", 4: "MAXITER", -1: "NOT_RUN"}


class DpgoError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"dpgo_b200 error {code}: {msg}")
        self.code = code


class OptParams(C.Structure):
    _fields_ = [("algorithm", C.c_int32), ("tr_iterations", C.c_int32), ("tr_max_inner", C.c_int32),
                ("precond", C.c_int32), ("rgd_stepsize", C.c_double), ("tr_tolerance", C.c_double),
                ("tr_initial_radius", C.c_double)]


class OptResult(C.Structure):
    _fields_ = [("success", C.c_int32), ("tcg_status", C.c_int32), ("tcg_iterations", C.c_int32),
                ("outer_iterations", C.c_int32), ("rejections", C.c_int32), ("spmv_passes", C.c_int32), ("precond_applies", C.c_int32),
                ("reserved0", C.c_int32),
                ("f_init", C.c_double), ("gradnorm_init", C.c_double), ("f_opt", C.c_double),
                ("gradnorm_opt", C.c_double), ("relative_change", C.c_double), ("elapsed_ms", C.c_double),
                ("quad_init", C.c_double), ("lin_init", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int32)
_vp = C.c_void_p

# name -> (restype, argtypes); every symbol include/dpgo_b200.h declares
SIGNATURES = {
    "dpgo_abi_version": (C.c_int, []),
    "dpgo_last_error": (C.c_char_p, []),
    "dpgo_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "dpgo_opt_params_default": (None, [C.POINTER(OptParams)]),
    "dpgo_problem_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_vp)]),
    "dpgo_problem_destroy": (C.c_int, [_vp]),
    "dpgo_problem_set_stream": (C.c_int, [_vp, _vp]),
    "dpgo_problem_sync": (C.c_int, [_vp]),
    "dpgo_problem_set_launch_mode": (C.c_int, [_vp, C.c_int]),
    "dpgo_problem_launch_info": (C.c_int, [_vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "dpgo_problem_dims": (C.c_int, [_vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                    C.POINTER(C.c_int64)]),
    "dpgo_problem_set_Q_csr": (C.c_int, [_vp, C.c_int, _ip, _ip, _dp, C.c_uint]),
    "dpgo_problem_set_Q_blocks": (C.c_int, [_vp, C.c_int64, _ip, _ip, _dp, C.c_uint]),
    "dpgo_problem_set_edges": (C.c_int, [_vp, C.c_int64, _ip, _ip, _dp, _dp, _dp, _dp, _dp, _ip, C.c_int64, _ip, _dp, C.c_uint]),
    "dpgo_problem_robust_reweight": (C.c_int, [_vp, C.c_int, C.c_double, C.c_double, _dp, _dp]),
    "dpgo_problem_set_edge_weights": (C.c_int, [_vp, _dp]),
    "dpgo_problem_set_edge_weights_async": (C.c_int, [_vp, _vp]),
    "dpgo_problem_robust_reweight_async": (C.c_int, [_vp, C.c_int, C.c_double, C.c_double]),
    "dpgo_problem_device_edge_weights": (C.c_int, [_vp, C.POINTER(_vp), C.POINTER(_vp)]),
    "dpgo_problem_gnc_counts": (C.c_int, [_vp, C.POINTER(C.c_int64)]),
    "dpgo_problem_set_G_dense": (C.c_int, [_vp, _dp]),
    "dpgo_problem_set_G_csr": (C.c_int, [_vp, _ip, _ip, _dp]),
    "dpgo_problem_f": (C.c_int, [_vp, _dp, _dp]),
    "dpgo_problem_egrad": (C.c_int, [_vp, _dp, _dp]),
    "dpgo_problem_ehess": (C.c_int, [_vp, _dp, _dp]),
    "dpgo_problem_rgrad": (C.c_int, [_vp, _dp, _dp, _dp]),
    "dpgo_problem_f_rgradnorm": (C.c_int, [_vp, _dp, _dp, _dp]),
    "dpgo_problem_rhess": (C.c_int, [_vp, _dp, _dp, _dp]),
    "dpgo_problem_precon": (C.c_int, [_vp, C.c_int, _dp, _dp, _dp]),
    "dpgo_manifold_tangent_project": (C.c_int, [_vp, _dp, _dp, _dp]),
    "dpgo_manifold_retract": (C.c_int, [_vp, _dp, _dp, _dp]),
    "dpgo_manifold_project": (C.c_int, [_vp, _dp, _dp]),
    "dpgo_optimize": (C.c_int, [_vp, C.POINTER(OptParams), _dp, _dp, C.POINTER(OptResult)]),
    "dpgo_problem_upload_X": (C.c_int, [_vp, _dp]),
    "dpgo_problem_download_X": (C.c_int, [_vp, _dp]),
    "dpgo_problem_upload_X_async": (C.c_int, [_vp, _dp]),
    "dpgo_problem_download_X_async": (C.c_int, [_vp, _dp]),
    "dpgo_problem_copy_X_from_device": (C.c_int, [_vp, _vp]),
    "dpgo_problem_device_X": (C.c_int, [_vp, C.POINTER(_vp)]),
    "dpgo_problem_device_G": (C.c_int, [_vp, C.POINTER(_vp)]),
    "dpgo_optimize_resident_async": (C.c_int, [_vp, C.POINTER(OptParams)]),
    "dpgo_optimize_result": (C.c_int, [_vp, C.POINTER(OptResult)]),
    "dpgo_spmv_device": (C.c_int, [_vp, _vp, _vp, C.c_int]),
    "dpgo_spmv_algorithmic_bytes": (C.c_int64, [_vp, C.c_int]),
    "dpgo_precond_algorithmic_bytes": (C.c_int64, [_vp, C.c_int]),
    "dpgo_nd_info": (C.c_int, [_vp, C.POINTER(C.c_int64)]),
    "dpgo_nd_node_sizes": (C.c_int, [_vp, C.c_int64, _ip, _ip, _ip, C.POINTER(C.c_int64)]),
    "dpgo_nd_debug_emulate": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int64, _ip, _ip, _dp, C.c_double, C.c_int, C.c_int,
                                        C.c_int, _dp, _dp, C.POINTER(C.c_int64)]),
    "dpgo_debug_phase_latency": (C.c_int, [_vp, C.c_int, _dp, _dp]),
    "dpgo_debug_phase_times64": (C.c_int, [_vp, C.c_int, _dp]),
    "dpgo_chordal_initialization": (C.c_int, [C.c_int, C.c_int, C.c_int64, _ip, _ip, _dp, _dp, _dp, _dp, C.c_int, C.c_double,
                                              C.c_int, _dp, _ip]),
    "dpgo_chordal_last_error": (C.c_char_p, []),
    "dpgo_pose_covariances": (C.c_int, [C.c_int, C.c_int, C.c_int64, _ip, _ip, _dp, _dp, _dp, _dp, _dp, _dp, C.c_int, C.c_int,
                                        C.c_int64, _ip, _dp, _dp, C.POINTER(C.c_int64)]),
    "dpgo_pose_covariances_debug_emulate": (C.c_int, [C.c_int, C.c_int, C.c_int64, _ip, _ip, _dp, _dp, _dp, _dp, _dp, _dp, C.c_int,
                                                      C.c_int, C.c_int, C.c_int64, _ip, _dp, _dp, C.POINTER(C.c_int64)]),
    "dpgo_device_set": (C.c_int, [C.c_int]),
    "dpgo_device_malloc": (C.c_int, [C.c_int, C.c_size_t, C.POINTER(_vp)]),
    "dpgo_device_free": (C.c_int, [C.c_int, _vp]),
    "dpgo_stream_create": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "dpgo_stream_destroy": (C.c_int, [C.c_int, _vp]),
    "dpgo_stream_synchronize": (C.c_int, [C.c_int, _vp]),
    "dpgo_agent_set_public_poses": (C.c_int, [_vp, C.c_int, _ip]),
    "dpgo_agent_pack_public": (C.c_int, [_vp, _vp]),
    "dpgo_agent_set_shared_edges": (C.c_int, [_vp, C.c_int, _ip, _ip, _ip, _dp, _dp]),
    "dpgo_agent_build_G": (C.c_int, [_vp, _vp, C.c_int64]),
    "dpgo_agent_accel_init": (C.c_int, [_vp]),
    "dpgo_agent_accel_begin": (C.c_int, [_vp, C.c_double]),
    "dpgo_agent_accel_end": (C.c_int, [_vp, C.c_double, C.c_int]),
    "dpgo_agent_accel_restart_begin": (C.c_int, [_vp]),
    "dpgo_agent_accel_restart_end": (C.c_int, [_vp]),
    "dpgo_agent_pack_public_aux": (C.c_int, [_vp, _vp]),
    "dpgo_agents_round_async": (C.c_int, [C.POINTER(_vp), C.c_int, C.POINTER(OptParams), _vp, C.c_int64, C.POINTER(_vp), _vp,
                                          C.c_int]),
    "dpgo_agents_accel_begin_async": (C.c_int, [C.POINTER(_vp), C.c_int, _ip, C.c_double, C.c_int, C.POINTER(_vp),
                                                C.POINTER(_vp), _vp]),
    "dpgo_agents_accel_round_async": (C.c_int, [C.POINTER(_vp), C.c_int, C.POINTER(OptParams), _vp, _vp, C.c_int64, _vp]),
    "dpgo_agent_accel_state": (C.c_int, [_vp, _dp]),
    "dpgo_agents_host_io_async": (C.c_int, [C.POINTER(_vp), C.c_int, C.POINTER(_vp), C.POINTER(_vp), C.c_int, _vp]),
    "dpgo_agent_f_rgradnorm_resident": (C.c_int, [_vp, _dp, _dp]),
    "dpgo_agent_set_local_trajectory": (C.c_int, [_vp, _dp, _dp]),
    "dpgo_agent_set_align_candidates": (C.c_int, [_vp, C.c_int, _ip, _ip, _ip, _ip, _ip, _dp]),
    "dpgo_agents_align_async": (C.c_int, [C.POINTER(_vp), C.c_int, _vp, C.c_int64, _ip, C.c_int, _vp]),
    "dpgo_agent_align_result": (C.c_int, [_vp, _dp, _ip]),
    "dpgo_robust_single_rotation_averaging": (C.c_int, [C.c_int, C.c_int, C.c_int, _dp, _dp, C.c_double, _dp, _ip, _ip]),
    "dpgo_agents_status_async": (C.c_int, [C.POINTER(_vp), C.c_int, _ip, _vp, _vp]),
    "dpgo_agent_trajectory_global": (C.c_int, [_vp, _dp, _dp]),
    "dpgo_host_alloc_pinned": (C.c_int, [C.c_size_t, C.POINTER(_vp)]),
    "dpgo_host_free_pinned": (C.c_int, [_vp]),
    "dpgo_copy_to_host_async": (C.c_int, [C.c_int, _vp, _vp, C.c_size_t, _vp]),
    "dpgo_agents_set_agent_graph": (C.c_int, [_vp, C.c_int, _ip, _ip]),
    "dpgo_agents_select_round_async": (C.c_int, [C.POINTER(_vp), C.c_int, _ip, C.POINTER(OptParams), _vp, _vp, C.c_int64,
                                                 C.POINTER(_vp), _vp]),
    "dpgo_agents_selection_log": (C.c_int, [_vp, C.c_int64, C.c_int64, C.POINTER(C.c_uint8), C.POINTER(C.c_int64)]),
}

_lib = None


def load_library(path: str | None = None) -> C.CDLL:
    """dlopen the in-tree library and bind every declared symbol (raises if one is missing)."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise DpgoError(-1, f"{path} not found: build it with `python -m dpo_b200.build` "
                            "(__graft_entry__.build()); there is no CPU fallback")
    lib = C.CDLL(path)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def last_error() -> str:
    return load_library().dpgo_last_error().decode("utf-8", "replace")


def check(code: int) -> None:
    if code != OK:
        raise DpgoError(code, last_error())


def dptr(a: np.ndarray):
    return a.ctypes.data_as(_dp)


def iptr(a: np.ndarray):
    return a.ctypes.data_as(_ip)


def as_colmajor(X: np.ndarray, r: int, N: int) -> np.ndarray:
    """Return X (shape (r, N)) as a Fortran-contiguous float64 array (the ABI's column-major layout)."""
    X = np.asarray(X, dtype=np.float64)
    if X.shape != (r, N):
        raise ValueError(f"expected shape {(r, N)}, got {X.shape}")
    return np.asfortranarray(X)

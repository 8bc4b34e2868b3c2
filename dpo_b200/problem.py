"""Python host mirror of the reference's QuadraticProblem / QuadraticOptimizer over the C ABI.

Same class and method names, argument meaning and error behaviour as the reference
(include/DPGO/QuadraticProblem.h:31-109, include/DPGO/QuadraticOptimizer.h:20-76) so the parity
tests read like the reference's own.  All numerics run in libdpgo_b200.so on the GPU.
Matrices are NumPy arrays of shape (r, (d+1) n); they are converted to the ABI's column-major
layout at the boundary.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _capi as capi
from ._capi import (ALG_RGD, ALG_RTR, PRECOND_BLOCK_JACOBI, PRECOND_DENSE_EXACT, PRECOND_NONE, PRECOND_SPARSE_EXACT,
                    OptParams, OptResult)


class _DeviceArray:
    """__cuda_array_interface__ of m float64 at a device address; keeps the owning problem alive while viewed."""

    def __init__(self, ptr: int, m: int, owner):
        self._owner = owner
        self.__cuda_array_interface__ = {"shape": (m,), "typestr": "<f8", "data": (ptr or 0, False), "version": 3,
                                         "strides": None, "stream": None}


def _device_view(ptr: int, m: int, device: int, owner):
    import torch
    t = torch.as_tensor(_DeviceArray(ptr, m, owner), device=torch.device("cuda", device))
    t._dpgo_owner = owner
    return t


class ROPTALG:
    """ref: include/DPGO/DPGO_types.h:29-35"""
    RTR = ALG_RTR
    RGD = ALG_RGD


class QuadraticProblem:
    """f(X) = 0.5 <Q, X^T X> + <X, G> on (St(d,r) x R^r)^n, resident on one GPU.

    ref: include/DPGO/QuadraticProblem.h:31-109, src/QuadraticProblem.cpp.
    """

    def __init__(self, n: int, d: int, r: int, device: int = 0,
                 preconditioners=(PRECOND_BLOCK_JACOBI, PRECOND_SPARSE_EXACT), cluster: bool = False):
        self._lib = capi.load_library()
        self.n, self.d, self.r = int(n), int(d), int(r)
        self.N = (self.d + 1) * self.n
        self.device = device
        self._precond_mask = 0
        for m in preconditioners:
            self._precond_mask |= 1 << m
        h = C.c_void_p()
        capi.check(self._lib.dpgo_problem_create(self.n, self.d, self.r, device, C.byref(h)))
        self._h = h
        if cluster:
            # the step kernel runs as ONE thread-block cluster, so that several small agents share the GPU
            capi.check(self._lib.dpgo_problem_set_launch_mode(self._h, 1))

    def launch_info(self):
        """(CTAs of the persistent step kernel, launched as one thread-block cluster?)"""
        g, c = C.c_int(), C.c_int()
        capi.check(self._lib.dpgo_problem_launch_info(self._h, C.byref(g), C.byref(c)))
        return g.value, bool(c.value)

    # -- lifetime --------------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.dpgo_problem_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- getters (ref .h:38-44) -----------------------------------------------------------------
    def num_poses(self) -> int:
        return self.n

    def dimension(self) -> int:
        return self.d

    def relaxation_rank(self) -> int:
        return self.r

    def num_blocks(self) -> int:
        nb = C.c_int64()
        capi.check(self._lib.dpgo_problem_dims(self._h, None, None, None, C.byref(nb)))
        return nb.value

    # -- cost matrices ---------------------------------------------------------------------------
    def setQ(self, Q, preconditioners=None) -> None:
        """Q: scipy.sparse matrix (any format) of shape ((d+1)n, (d+1)n).  ref: setQ, .cpp:31-42."""
        import scipy.sparse as sp
        if preconditioners is not None:
            self._precond_mask = 0
            for m in preconditioners:
                self._precond_mask |= 1 << m
        Q = sp.csr_matrix(Q)
        if Q.shape != (self.N, self.N):
            raise ValueError(f"Q must be {(self.N, self.N)}, got {Q.shape}")
        Q.sort_indices()
        rowptr = np.ascontiguousarray(Q.indptr, dtype=np.int32)
        colind = np.ascontiguousarray(Q.indices, dtype=np.int32)
        val = np.ascontiguousarray(Q.data, dtype=np.float64)
        capi.check(self._lib.dpgo_problem_set_Q_csr(self._h, self.N, capi.iptr(rowptr), capi.iptr(colind),
                                                    capi.dptr(val), self._precond_mask))

    def setQ_blocks(self, brow, bcol, blocks, preconditioners=None) -> None:
        """Block triplets: blocks[k] is the (d+1)x(d+1) sub-matrix of Q at (brow[k], bcol[k])."""
        if preconditioners is not None:
            self._precond_mask = 0
            for m in preconditioners:
                self._precond_mask |= 1 << m
        dh = self.d + 1
        brow = np.ascontiguousarray(brow, dtype=np.int32)
        bcol = np.ascontiguousarray(bcol, dtype=np.int32)
        blocks = np.ascontiguousarray(blocks, dtype=np.float64).reshape(-1, dh, dh)
        if not (brow.shape[0] == bcol.shape[0] == blocks.shape[0]):
            raise ValueError("block triplet arrays disagree in length")
        capi.check(self._lib.dpgo_problem_set_Q_blocks(self._h, brow.shape[0], capi.iptr(brow), capi.iptr(bcol),
                                                       capi.dptr(blocks), self._precond_mask))

    ROBUST = {"L2": 0, "L1": 1, "Huber": 2, "TLS": 3, "GM": 4, "GNC_TLS": 5}

    def setEdges(self, edges, static_pose=None, static_blocks=None, fixed=None, preconditioners=None) -> None:
        """Q assembled on the device from raw edge records (ref constructConnectionLaplacianSE, src/DPGO_utils.cpp:199-271;
        diagonal terms of PGOAgent::constructQMatrix, src/PGOAgent.cpp:746-775 as `static` blocks at (pose, pose)).
        `edges`: posegraph.EdgeSet with local pose ids; `fixed`: per-edge flags whose weights robustReweight leaves alone."""
        if preconditioners is not None:
            self._precond_mask = 0
            for m in preconditioners:
                self._precond_mask |= 1 << m
        dh = self.d + 1
        p1 = np.ascontiguousarray(edges.p1, dtype=np.int32)
        p2 = np.ascontiguousarray(edges.p2, dtype=np.int32)
        R = np.ascontiguousarray(edges.R, dtype=np.float64)
        t = np.ascontiguousarray(edges.t, dtype=np.float64)
        ka = np.ascontiguousarray(edges.kappa, dtype=np.float64)
        ta = np.ascontiguousarray(edges.tau, dtype=np.float64)
        w = np.ascontiguousarray(edges.weight, dtype=np.float64)
        fx = None if fixed is None else np.ascontiguousarray(fixed, dtype=np.int32)
        ns = 0 if static_pose is None else len(static_pose)
        sp_ = None if ns == 0 else np.ascontiguousarray(static_pose, dtype=np.int32)
        sb_ = None if ns == 0 else np.ascontiguousarray(static_blocks, dtype=np.float64).reshape(ns, dh, dh)
        capi.check(self._lib.dpgo_problem_set_edges(
            self._h, len(p1), capi.iptr(p1), capi.iptr(p2), capi.dptr(R), capi.dptr(t), capi.dptr(ka), capi.dptr(ta), capi.dptr(w),
            None if fx is None else capi.iptr(fx), ns, None if sp_ is None else capi.iptr(sp_),
            None if sb_ is None else capi.dptr(sb_), self._precond_mask))
        self._num_edges = len(p1)

    def robustReweight(self, cost: str, mu: float = 1.0, param: float = 1.0):
        """Weights of the non-fixed edges at the RESIDENT iterate (upload_X first), Q re-assembled on the device.
        ref PGOAgent::updateLoopClosuresWeights, src/PGOAgent.cpp:1181-1245.  Returns (weights, squared residuals)."""
        m = getattr(self, "_num_edges", 0)
        w, r2 = np.zeros(max(m, 1)), np.zeros(max(m, 1))
        capi.check(self._lib.dpgo_problem_robust_reweight(self._h, self.ROBUST[cost], float(mu), float(param), capi.dptr(w), capi.dptr(r2)))
        return w[:m], r2[:m]

    def setEdgeWeights(self, weights) -> None:
        w = np.ascontiguousarray(weights, dtype=np.float64)
        capi.check(self._lib.dpgo_problem_set_edge_weights(self._h, capi.dptr(w)))

    # -- stream-ordered re-weighting (no host copy, no synchronisation; see dpgo_problem_robust_reweight_async) ---------
    def robustReweightAsync(self, cost: str, mu: float = 1.0, param: float = 1.0) -> None:
        """robustReweight on the handle's stream: weights, Q and the prepared preconditioners all refreshed on the device.
        The first call after setEdges builds the sparse exact preconditioner's structure on the host and synchronises;
        every later one can be captured into a CUDA graph."""
        capi.check(self._lib.dpgo_problem_robust_reweight_async(self._h, self.ROBUST[cost], float(mu), float(param)))

    def setEdgeWeightsAsync(self, weights) -> None:
        """weights: a float64 CUDA tensor of the edge count on the problem's device, or a device pointer (int).  Read in
        the handle's stream order."""
        if isinstance(weights, int):
            ptr = weights
        else:
            if not (getattr(weights, "is_cuda", False) and weights.dtype.is_floating_point and weights.element_size() == 8):
                raise ValueError("weights must be a float64 CUDA tensor or a device pointer")
            if weights.device.index != self.device or weights.numel() != getattr(self, "_num_edges", 0) or not weights.is_contiguous():
                raise ValueError("weights must be a contiguous tensor of one weight per edge on the problem's device")
            ptr = weights.data_ptr()
        capi.check(self._lib.dpgo_problem_set_edge_weights_async(self._h, C.c_void_p(ptr)))

    def edgeWeightsDevice(self):
        """(weights, squared residuals): torch float64 views of the device arrays (one entry per edge), not copies."""
        import torch
        w, r2 = C.c_void_p(), C.c_void_p()
        capi.check(self._lib.dpgo_problem_device_edge_weights(self._h, C.byref(w), C.byref(r2)))
        m = getattr(self, "_num_edges", 0)
        return _device_view(w.value, m, self.device, self), _device_view(r2.value, m, self.device, self)

    def gncCounts(self):
        """(weight 1, weight 0, in between) over the non-fixed edges at the last re-weight (synchronises)."""
        out = (C.c_int64 * 3)()
        capi.check(self._lib.dpgo_problem_gnc_counts(self._h, out))
        return int(out[0]), int(out[1]), int(out[2])

    def nd_node_sizes(self):
        """(own poses, boundary poses, stage) of every macro node of the sparse exact preconditioner (prepares it)."""
        cnt = C.c_int64()
        capi.check(self._lib.dpgo_nd_node_sizes(self._h, 0, None, None, None, C.byref(cnt)))
        own, bnd, st = (np.zeros(max(cnt.value, 1), dtype=np.int32) for _ in range(3))
        capi.check(self._lib.dpgo_nd_node_sizes(self._h, cnt.value, capi.iptr(own), capi.iptr(bnd), capi.iptr(st), C.byref(cnt)))
        n = cnt.value
        return own[:n], bnd[:n], st[:n]

    def setG(self, G) -> None:
        """G: dense (r, (d+1)n) array, scipy sparse matrix, or None to clear.  ref: setG, .cpp:44-48."""
        if G is None:
            capi.check(self._lib.dpgo_problem_set_G_dense(self._h, None))
            return
        if hasattr(G, "toarray"):
            G = G.toarray()
        Gf = capi.as_colmajor(G, self.r, self.N)
        capi.check(self._lib.dpgo_problem_set_G_dense(self._h, capi.dptr(Gf)))

    # -- evaluation --------------------------------------------------------------------------------
    def _in(self, X):
        return capi.as_colmajor(X, self.r, self.N)

    def _out(self):
        return np.empty((self.r, self.N), dtype=np.float64, order="F")

    def f(self, Y) -> float:
        out = C.c_double()
        Yf = self._in(Y)
        capi.check(self._lib.dpgo_problem_f(self._h, capi.dptr(Yf), C.byref(out)))
        return out.value

    def EucGrad(self, X) -> np.ndarray:
        Xf, out = self._in(X), self._out()
        capi.check(self._lib.dpgo_problem_egrad(self._h, capi.dptr(Xf), capi.dptr(out)))
        return out

    def EucHessianEta(self, V) -> np.ndarray:
        Vf, out = self._in(V), self._out()
        capi.check(self._lib.dpgo_problem_ehess(self._h, capi.dptr(Vf), capi.dptr(out)))
        return out

    def RieGrad(self, Y) -> np.ndarray:
        Yf, out = self._in(Y), self._out()
        capi.check(self._lib.dpgo_problem_rgrad(self._h, capi.dptr(Yf), capi.dptr(out), None))
        return out

    def RieGradNorm(self, Y) -> float:
        nrm = C.c_double()
        Yf = self._in(Y)
        capi.check(self._lib.dpgo_problem_rgrad(self._h, capi.dptr(Yf), None, C.byref(nrm)))
        return nrm.value

    def f_and_gradnorm(self, Y):
        fo, nrm = C.c_double(), C.c_double()
        Yf = self._in(Y)
        capi.check(self._lib.dpgo_problem_f_rgradnorm(self._h, capi.dptr(Yf), C.byref(fo), C.byref(nrm)))
        return fo.value, nrm.value

    def RieHessianEta(self, X, V) -> np.ndarray:
        Xf, Vf, out = self._in(X), self._in(V), self._out()
        capi.check(self._lib.dpgo_problem_rhess(self._h, capi.dptr(Xf), capi.dptr(Vf), capi.dptr(out)))
        return out

    def PreConditioner(self, X, V, precond: int = PRECOND_SPARSE_EXACT) -> np.ndarray:
        Xf, Vf, out = self._in(X), self._in(V), self._out()
        capi.check(self._lib.dpgo_problem_precon(self._h, precond, capi.dptr(Xf), capi.dptr(Vf), capi.dptr(out)))
        return out

    # -- manifold ------------------------------------------------------------------------------------
    def Projection(self, X, Z) -> np.ndarray:
        Xf, Zf, out = self._in(X), self._in(Z), self._out()
        capi.check(self._lib.dpgo_manifold_tangent_project(self._h, capi.dptr(Xf), capi.dptr(Zf), capi.dptr(out)))
        return out

    def Retraction(self, X, eta) -> np.ndarray:
        Xf, Ef, out = self._in(X), self._in(eta), self._out()
        capi.check(self._lib.dpgo_manifold_retract(self._h, capi.dptr(Xf), capi.dptr(Ef), capi.dptr(out)))
        return out

    def project(self, M) -> np.ndarray:
        """ref: LiftedSEManifold::project, src/manifold/LiftedSEManifold.cpp:34-45."""
        Mf, out = self._in(M), self._out()
        capi.check(self._lib.dpgo_manifold_project(self._h, capi.dptr(Mf), capi.dptr(out)))
        return out

    # -- device-resident path ----------------------------------------------------------------------------
    def set_stream(self, cuda_stream: Optional[int]) -> None:
        """cuda_stream: a cudaStream_t handle; 0 means the legacy default stream (torch's default), None
        restores the handle's own non-blocking stream."""
        if cuda_stream is None:
            arg = None
        elif cuda_stream == 0:
            arg = C.c_void_p(1)                      # cudaStreamLegacy
        else:
            arg = C.c_void_p(cuda_stream)
        capi.check(self._lib.dpgo_problem_set_stream(self._h, arg))

    def sync(self) -> None:
        capi.check(self._lib.dpgo_problem_sync(self._h))

    def upload_X(self, X) -> None:
        Xf = self._in(X)
        capi.check(self._lib.dpgo_problem_upload_X(self._h, capi.dptr(Xf)))

    def download_X(self) -> np.ndarray:
        out = self._out()
        capi.check(self._lib.dpgo_problem_download_X(self._h, capi.dptr(out)))
        return out

    def upload_X_async(self, Xf: np.ndarray) -> None:
        """Xf: Fortran-contiguous (r, N) float64 (pinned for a truly asynchronous copy); no synchronisation."""
        capi.check(self._lib.dpgo_problem_upload_X_async(self._h, capi.dptr(Xf)))

    def download_X_async(self, out: np.ndarray) -> None:
        capi.check(self._lib.dpgo_problem_download_X_async(self._h, capi.dptr(out)))

    def copy_X_from_device(self, src_ptr: int) -> None:
        capi.check(self._lib.dpgo_problem_copy_X_from_device(self._h, C.c_void_p(src_ptr)))

    def device_X_ptr(self) -> int:
        p = C.c_void_p()
        capi.check(self._lib.dpgo_problem_device_X(self._h, C.byref(p)))
        return p.value

    def device_G_ptr(self) -> int:
        p = C.c_void_p()
        capi.check(self._lib.dpgo_problem_device_G(self._h, C.byref(p)))
        return p.value

    def spmv_device(self, x_ptr: int, out_ptr: int, add_G: bool = False) -> None:
        capi.check(self._lib.dpgo_spmv_device(self._h, C.c_void_p(x_ptr), C.c_void_p(out_ptr), int(add_G)))

    def spmv_algorithmic_bytes(self, add_G: bool = False) -> int:
        return int(self._lib.dpgo_spmv_algorithmic_bytes(self._h, int(add_G)))

    def nd_ready(self) -> bool:
        """True once the sparse exact preconditioner was requested for this problem (its hierarchy can be queried)."""
        return bool(self._precond_mask & (1 << PRECOND_SPARSE_EXACT))

    def nd_info(self) -> dict:
        """Diagnostics of the sparse exact preconditioner's hierarchy (prepares it if needed)."""
        info = (C.c_int64 * 16)()
        capi.check(self._lib.dpgo_nd_info(self._h, info))
        keys = ("levels", "nodes", "phases", "block_bytes", "bytes_per_apply", "max_own", "max_bnd", "nd_depth", "steps",
                "jobs", "epilogues", "max_ytiles", "max_slots", "resident_bytes", "max_resident_bytes_per_cta")
        out = {k: int(info[i]) for i, k in enumerate(keys)}
        # share of the panel bytes of an application read from shared memory (every application of a launch but the first)
        out["resident_fraction"] = out["resident_bytes"] / max(out["bytes_per_apply"], 1)
        return out

    def precond_algorithmic_bytes(self, preconditioner: int) -> int:
        return int(self._lib.dpgo_precond_algorithmic_bytes(self._h, int(preconditioner)))

    def resident_f_gradnorm(self):
        fo, nrm = C.c_double(), C.c_double()
        capi.check(self._lib.dpgo_agent_f_rgradnorm_resident(self._h, C.byref(fo), C.byref(nrm)))
        return fo.value, nrm.value


class QuadraticOptimizer:
    """ref: include/DPGO/QuadraticOptimizer.h:20-76, src/QuadraticOptimizer.cpp:20-149."""

    def __init__(self, problem: QuadraticProblem):
        self.problem = problem
        self._lib = problem._lib
        self._p = OptParams()
        self._lib.dpgo_opt_params_default(C.byref(self._p))
        self.verbose = False
        self.result = OptResult()

    def setProblem(self, p: QuadraticProblem) -> None:
        self.problem = p

    def setVerbose(self, v: bool) -> None:
        self.verbose = bool(v)

    def setAlgorithm(self, alg: int) -> None:
        self._p.algorithm = int(alg)

    def setGradientDescentStepsize(self, s: float) -> None:
        self._p.rgd_stepsize = float(s)

    def setTrustRegionIterations(self, it: int) -> None:
        self._p.tr_iterations = int(it)

    def setTrustRegionTolerance(self, tol: float) -> None:
        self._p.tr_tolerance = float(tol)

    def setTrustRegionInitialRadius(self, radius: float) -> None:
        self._p.tr_initial_radius = float(radius)

    def setTrustRegionMaxInnerIterations(self, it: int) -> None:
        self._p.tr_max_inner = int(it)

    def setPreconditioner(self, precond: int) -> None:
        """GPU extension: SPARSE_EXACT (reference operator, nested-dissection block solve; default) |
        DENSE_EXACT (same operator through a dense inverse, A/B) | BLOCK_JACOBI (throughput) | NONE."""
        self._p.precond = int(precond)

    def params(self) -> OptParams:
        return self._p

    def optimize(self, Y, out: Optional[np.ndarray] = None) -> np.ndarray:
        """One optimize() call, host in / host out.  `out` may be a caller-owned (e.g. pinned) Fortran-ordered
        (r, (d+1)n) float64 array that receives the result."""
        pr = self.problem
        Yf = pr._in(Y)
        if out is None:
            out = pr._out()
        elif out.shape != (pr.r, pr.N) or out.dtype != np.float64 or not out.flags.f_contiguous:
            raise ValueError("out must be a Fortran-contiguous float64 array of shape (r, (d+1)n)")
        capi.check(self._lib.dpgo_optimize(pr._h, C.byref(self._p), capi.dptr(Yf), capi.dptr(out),
                                           C.byref(self.result)))
        if self.verbose:
            print(f"[dpgo_b200] f {self.result.f_init:.10g} -> {self.result.f_opt:.10g}, "
                  f"|g| {self.result.gradnorm_init:.6g} -> {self.result.gradnorm_opt:.6g}, "
                  f"tCG {capi.TCG_NAMES.get(self.result.tcg_status)} x{self.result.tcg_iterations}")
        return out

    # resident variants: iterate stays in HBM
    def optimize_resident_async(self) -> None:
        capi.check(self._lib.dpgo_optimize_resident_async(self.problem._h, C.byref(self._p)))

    def fetch_result(self) -> OptResult:
        capi.check(self._lib.dpgo_optimize_result(self.problem._h, C.byref(self.result)))
        return OptResult.from_buffer_copy(self.result)

    def getOptResult(self) -> OptResult:
        return self.result

    def problem_stats(self):
        """(<XQ,X>, <X,G>, |rgrad|^2, f) of the resident iterate -- per-agent inputs of the central trace."""
        fo, nrm = C.c_double(), C.c_double()
        capi.check(self._lib.dpgo_agent_f_rgradnorm_resident(self.problem._h, C.byref(fo), C.byref(nrm)))
        st = OptResult()
        capi.check(self._lib.dpgo_optimize_result(self.problem._h, C.byref(st)))
        return (st.quad_init, st.lin_init, nrm.value ** 2, fo.value)

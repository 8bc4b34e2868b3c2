"""CPU oracle for the distributed pose-graph-optimisation hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is part of the product: only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may import
it, and only as the checker.  The product path is the CUDA library behind
``include/dpgo_b200.h``.

This module restates, in NumPy/SciPy, the algorithm the reference (tjcunhao/dpo, a fork of
mit-acl/dpgo) runs on the CPU through Eigen + CHOLMOD + ROPTLIB.  The reference cannot be
built in this image (Eigen, SuiteSparse, ROPTLIB, Boost absent, no network), so parity is
PINNED instead against the reference's own shipped artefacts (``tests/test_oracle_golden.py``):
  * ``result/graph/NP<dataset>.txt`` per-iteration ``2f, |grad|`` traces (5 agents, r=5, RTR),
  * ``vis.ipynb:108746,108748`` chordal-initialisation cost / gradient-norm constants,
  * ``tests/testTriangleGraph.cpp:15-29`` known-answer fixture.

Reference lines each function follows are cited as ``ref: <file>:<lines>`` (paths relative to
the reference root).  ROPTLIB (third party, not vendored; ``cmake/roptlib.cmake:7-8``,
``yuluntian/ROPTLIB`` branch ``feature/cmake``, no pinned commit) arithmetic is restated from
its published algorithm (Absil/Baker/Gallivan RTR with Steihaug-Toint truncated CG) and
anchored on the reference call sites ``src/QuadraticOptimizer.cpp:61-149``.

Array convention: a point ``X`` is a NumPy array of shape ``(r, (d+1)*n)``; pose ``i``
occupies columns ``[(d+1)i, (d+1)(i+1))`` (rotation-like ``r x d`` block ``Y_i`` then the
translation-like column ``p_i``) exactly as in the reference's column-major Eigen matrix.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla


# --------------------------------------------------------------------------------------
# Measurements and the g2o reader
# --------------------------------------------------------------------------------------
@dataclass
class Measurements:
    """Struct-of-arrays view of a list of relative SE(d) measurements.

    ref: include/DPGO/RelativeSEMeasurement.h:21-50 (fields r1,r2,p1,p2,R,t,kappa,tau,weight)
    """
    d: int
    r1: np.ndarray
    r2: np.ndarray
    p1: np.ndarray
    p2: np.ndarray
    R: np.ndarray       # (m, d, d)
    t: np.ndarray       # (m, d)
    kappa: np.ndarray
    tau: np.ndarray
    weight: np.ndarray

    def __len__(self) -> int:
        return int(self.p1.shape[0])

    def subset(self, idx) -> "Measurements":
        idx = np.asarray(idx, dtype=np.int64)
        return Measurements(self.d, self.r1[idx], self.r2[idx], self.p1[idx], self.p2[idx],
                            self.R[idx], self.t[idx], self.kappa[idx], self.tau[idx],
                            self.weight[idx])

    @staticmethod
    def empty(d: int) -> "Measurements":
        z = np.zeros(0, dtype=np.int64)
        return Measurements(d, z, z.copy(), z.copy(), z.copy(), np.zeros((0, d, d)),
                            np.zeros((0, d)), np.zeros(0), np.zeros(0), np.zeros(0))

    @staticmethod
    def concat(parts: Sequence["Measurements"]) -> "Measurements":
        d = parts[0].d
        cat = lambda name: np.concatenate([getattr(p, name) for p in parts], axis=0)
        return Measurements(d, cat("r1"), cat("r2"), cat("p1"), cat("p2"), cat("R"), cat("t"),
                            cat("kappa"), cat("tau"), cat("weight"))


def quat_to_rot_unnormalised(w: float, x: float, y: float, z: float) -> np.ndarray:
    """Quaternion -> matrix WITHOUT normalising, as Eigen's ``toRotationMatrix`` does.

    ref: src/DPGO_utils.cpp:160 (``Eigen::Quaterniond(dqw,dqx,dqy,dqz).toRotationMatrix()``).
    Normalising first shifts the golden traces by ~1e-8 relative.
    """
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1.0 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1.0 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1.0 - (txx + tyy)]])


def read_g2o(path: str) -> Tuple[Measurements, int]:
    """Parse a .g2o file into measurements + pose count.  ref: src/DPGO_utils.cpp:64-197."""
    p1, p2, Rs, ts, kap, tau = [], [], [], [], [], []
    d = 0
    with open(path, "r") as fh:
        for line in fh:
            tok = line.split()
            if not tok:
                continue
            tag = tok[0]
            if tag == "EDGE_SE2":                                   # ref :96-126
                i, j = int(tok[1]), int(tok[2])
                dx, dy, dth = (float(v) for v in tok[3:6])
                I11, I12, I13, I22, I23, I33 = (float(v) for v in tok[6:12])
                d = 2
                c, s = math.cos(dth), math.sin(dth)
                Rs.append(np.array([[c, -s], [s, c]]))
                ts.append(np.array([dx, dy]))
                tran = np.array([[I11, I12], [I12, I22]])
                tau.append(2.0 / np.trace(np.linalg.inv(tran)))
                kap.append(I33)
            elif tag == "EDGE_SE3:QUAT":                            # ref :128-178
                i, j = int(tok[1]), int(tok[2])
                v = [float(q) for q in tok[3:31]]
                dx, dy, dz, qx, qy, qz, qw = v[0:7]
                (I11, I12, I13, I14, I15, I16, I22, I23, I24, I25, I26, I33, I34, I35, I36,
                 I44, I45, I46, I55, I56, I66) = v[7:28]
                d = 3
                Rs.append(quat_to_rot_unnormalised(qw, qx, qy, qz))
                ts.append(np.array([dx, dy, dz]))
                tran = np.array([[I11, I12, I13], [I12, I22, I23], [I13, I23, I33]])
                rot = np.array([[I44, I45, I46], [I45, I55, I56], [I46, I56, I66]])
                tau.append(3.0 / np.trace(np.linalg.inv(tran)))
                kap.append(3.0 / (2.0 * np.trace(np.linalg.inv(rot))))
            elif tag in ("VERTEX_SE2", "VERTEX_SE3:QUAT"):
                continue
            else:
                raise ValueError(f"unrecognised g2o record: {tag}")
            p1.append(i)
            p2.append(j)
    m = len(p1)
    p1a = np.asarray(p1, dtype=np.int64)
    p2a = np.asarray(p2, dtype=np.int64)
    num_poses = int(max(p1a.max(), p2a.max())) + 1 if m else 1
    meas = Measurements(d, np.zeros(m, np.int64), np.zeros(m, np.int64), p1a, p2a,
                        np.asarray(Rs).reshape(m, d, d), np.asarray(ts).reshape(m, d),
                        np.asarray(kap, dtype=float), np.asarray(tau, dtype=float), np.ones(m))
    return meas, num_poses


# --------------------------------------------------------------------------------------
# Connection Laplacian Q  (ref: src/DPGO_utils.cpp:199-271)
# --------------------------------------------------------------------------------------
def _homogeneous(meas: Measurements) -> np.ndarray:
    m, d = len(meas), meas.d
    T = np.zeros((m, d + 1, d + 1))
    T[:, :d, :d] = meas.R
    T[:, :d, d] = meas.t
    T[:, d, d] = 1.0
    return T


def _omega(meas: Measurements) -> np.ndarray:
    m, d = len(meas), meas.d
    Om = np.zeros((m, d + 1))
    Om[:, :d] = (meas.weight * meas.kappa)[:, None]
    Om[:, d] = meas.weight * meas.tau
    return Om


def laplacian_blocks(meas: Measurements, n: int):
    """Block triplets (row pose, col pose, (d+1)x(d+1) block) of ``Q = A Omega A^T``.

    Per edge (i -> j, T=[R t;0 1], Omega=diag(w*kappa.., w*tau)):
    ``Q_ii += T Om T^T``, ``Q_jj += Om``, ``Q_ij = -T Om``, ``Q_ji = -Om T^T``.
    ref: src/DPGO_utils.cpp:232-258 (A(i,k) = -T, A(j,k) = +I) and :264-271 (A*Omega*A^T).
    """
    T = _homogeneous(meas)
    Om = _omega(meas)
    TO = T * Om[:, None, :]                       # T * diag(Om)
    Wii = np.einsum("mab,mcb->mac", TO, T)        # T Om T^T
    Wjj = np.zeros_like(T)
    dh = meas.d + 1
    Wjj[:, np.arange(dh), np.arange(dh)] = Om
    rows = np.concatenate([meas.p1, meas.p2, meas.p1, meas.p2])
    cols = np.concatenate([meas.p1, meas.p2, meas.p2, meas.p1])
    blocks = np.concatenate([Wii, Wjj, -TO, -np.transpose(TO, (0, 2, 1))], axis=0)
    return rows, cols, blocks


def blocks_to_csr(rows, cols, blocks, n: int, dh: int) -> sp.csr_matrix:
    """Assemble block triplets into a scalar CSR matrix (duplicates summed)."""
    nb = rows.shape[0]
    rr = (rows[:, None, None] * dh + np.arange(dh)[None, :, None]) + np.zeros((1, 1, dh), np.int64)
    cc = (cols[:, None, None] * dh + np.arange(dh)[None, None, :]) + np.zeros((1, dh, 1), np.int64)
    Q = sp.coo_matrix((blocks.reshape(-1), (rr.reshape(-1), cc.reshape(-1))),
                      shape=(n * dh, n * dh)).tocsr()
    Q.sum_duplicates()
    Q.sort_indices()
    return Q


def construct_connection_laplacian(meas: Measurements, n: Optional[int] = None) -> sp.csr_matrix:
    """ref: src/DPGO_utils.cpp:264-271 ``constructConnectionLaplacianSE``."""
    if n is None:
        n = int(max(meas.p1.max(), meas.p2.max())) + 1 if len(meas) else 1
    rows, cols, blocks = laplacian_blocks(meas, n)
    return blocks_to_csr(rows, cols, blocks, n, meas.d + 1)


# --------------------------------------------------------------------------------------
# Small dense helpers
# --------------------------------------------------------------------------------------
def project_to_rotation_group(M: np.ndarray) -> np.ndarray:
    """ref: src/DPGO_utils.cpp:463-477."""
    U, _, Vt = np.linalg.svd(M)
    if np.linalg.det(U) * np.linalg.det(Vt) > 0:
        return U @ Vt
    U = U.copy()
    U[:, -1] *= -1.0
    return U @ Vt


def project_to_stiefel(M: np.ndarray) -> np.ndarray:
    """ref: src/DPGO_utils.cpp:479-485 (thin SVD, U V^T)."""
    U, _, Vt = np.linalg.svd(M, full_matrices=False)
    return U @ Vt


def fixed_stiefel_variable(d: int, r: int) -> np.ndarray:
    """A fixed element of St(d, r) used as the lifting matrix ``YLift``.

    ref: src/DPGO_utils.cpp:487-492 draws it from ROPTLIB's ``RandInManifold`` after
    ``srand(1)``; that value depends on glibc ``rand`` + ROPTLIB internals and is unpinned by
    any reference test beyond orthonormality/repeatability (tests/testUtils.cpp:12-25).  Cost,
    gradient norm and the whole RBCD trajectory are invariant/equivariant under the choice, so
    the oracle (and the product) use a deterministic QR of a fixed seeded Gaussian matrix.
    """
    rng = np.random.RandomState(1)
    A = rng.standard_normal((r, d))
    Qm, Rm = np.linalg.qr(A)
    Qm = Qm * np.sign(np.diag(Rm))[None, :]
    return Qm


# --------------------------------------------------------------------------------------
# Chordal initialisation  (ref: src/DPGO_utils.cpp:273-409, 434-461)
# --------------------------------------------------------------------------------------
def _lstsq_normal(A: sp.spmatrix, b: np.ndarray) -> np.ndarray:
    """min |A x - b| through the normal equations + two refinement steps (stand-in for SPQR)."""
    A = A.tocsc()
    AtA = (A.T @ A).tocsc()
    lu = spla.splu(AtA)
    x = lu.solve(A.T @ b)
    for _ in range(2):
        x = x + lu.solve(A.T @ (b - A @ x))
    return x


def chordal_initialization(meas: Measurements, n: int) -> np.ndarray:
    """SE-Sync style chordal relaxation.  Returns ``T`` of shape (d, (d+1) n).

    ref: src/DPGO_utils.cpp:273-360 (B1,B2,B3), :362-409 (rotations then translations),
    :434-461 (recoverTranslations).
    """
    d, m = meas.d, len(meas)
    d2 = d * d
    i, j = meas.p1, meas.p2
    e = np.arange(m)
    sqt = np.sqrt(meas.tau)
    sqk = np.sqrt(meas.kappa)
    # B1 (ref :296-318): rows e*d+l; -sqrt(tau) at i*d+l, +sqrt(tau) at j*d+l
    l = np.arange(d)
    r_b1 = (e[:, None] * d + l[None, :]).ravel()
    B1 = sp.coo_matrix((np.concatenate([np.repeat(-sqt, d), np.repeat(sqt, d)]),
                        (np.concatenate([r_b1, r_b1]),
                         np.concatenate([(i[:, None] * d + l[None, :]).ravel(),
                                         (j[:, None] * d + l[None, :]).ravel()]))),
                       shape=(d * m, d * n)).tocsr()
    # B2 (ref :320-334): entry (d e + r, d2 i + d k + r) = -sqrt(tau) t(k)
    k_idx, r_idx = np.meshgrid(np.arange(d), np.arange(d), indexing="ij")
    rows = (e[:, None, None] * d + r_idx[None]).ravel()
    cols = (i[:, None, None] * d2 + d * k_idx[None] + r_idx[None]).ravel()
    vals = (-sqt[:, None, None] * meas.t[:, :, None] * np.ones((1, 1, d))).ravel()
    B2 = sp.coo_matrix((vals, (rows, cols)), shape=(d * m, d2 * n)).tocsr()
    # B3 (ref :336-360): (e d2 + d r + l, i d2 + d c + l) = -sqrt(kappa) R(c, r);  (e d2 + l, j d2 + l) = sqrt(kappa)
    rr, cc, ll = np.meshgrid(np.arange(d), np.arange(d), np.arange(d), indexing="ij")
    rows3 = (e[:, None, None, None] * d2 + d * rr[None] + ll[None]).ravel()
    cols3 = (i[:, None, None, None] * d2 + d * cc[None] + ll[None]).ravel()
    Rcr = np.transpose(meas.R, (0, 2, 1))          # Rcr[m, r, c] = R[m, c, r]
    vals3 = (-sqk[:, None, None, None] * Rcr[:, :, :, None] * np.ones((1, 1, 1, d))).ravel()
    l2 = np.arange(d2)
    rows3b = (e[:, None] * d2 + l2[None, :]).ravel()
    cols3b = (j[:, None] * d2 + l2[None, :]).ravel()
    B3 = sp.coo_matrix((np.concatenate([vals3, np.repeat(sqk, d2)]),
                        (np.concatenate([rows3, rows3b]), np.concatenate([cols3, cols3b]))),
                       shape=(d2 * m, d2 * n)).tocsc()
    # rotations (ref :374-392): fix R_0 = I, least squares for the rest, project each block
    Id_vec = np.eye(d).reshape(-1, order="F")
    cR = B3[:, :d2] @ Id_vec
    rvec = -_lstsq_normal(B3[:, d2:], cR)
    Rch = np.zeros((d, d * n))
    Rch[:, :d] = np.eye(d)
    Rch[:, d:] = rvec.reshape(d, (n - 1) * d, order="F")
    for p in range(1, n):
        Rch[:, p * d:(p + 1) * d] = project_to_rotation_group(Rch[:, p * d:(p + 1) * d])
    # translations (ref :434-461)
    c = B2 @ Rch.reshape(-1, order="F")
    tred = -_lstsq_normal(B1.tocsc()[:, d:], c)
    tch = np.zeros((d, n))
    tch[:, 1:] = tred.reshape(d, n - 1, order="F")
    T = np.zeros((d, (d + 1) * n))
    for p in range(n):
        T[:, p * (d + 1):p * (d + 1) + d] = Rch[:, p * d:(p + 1) * d]
        T[:, p * (d + 1) + d] = tch[:, p]
    return T


def odometry_initialization(odom: Measurements, n: int) -> np.ndarray:
    """ref: src/DPGO_utils.cpp:411-432."""
    d = odom.d
    T = np.zeros((d, (d + 1) * n))
    T[:, :d] = np.eye(d)
    for s in range(len(odom)):
        assert odom.p1[s] == s and odom.p2[s] == s + 1
        Rs = T[:, s * (d + 1):s * (d + 1) + d]
        ts = T[:, s * (d + 1) + d]
        T[:, (s + 1) * (d + 1):(s + 1) * (d + 1) + d] = Rs @ odom.R[s]
        T[:, (s + 1) * (d + 1) + d] = ts + Rs @ odom.t[s]
    return T


# --------------------------------------------------------------------------------------
# Manifold (St(d,r) x R^r)^n  -- ROPTLIB semantics (ChooseStieParamsSet3: Euclidean metric,
# QF retraction, extrinsic representation; ref: src/manifold/LiftedSEManifold.cpp:16-24)
# --------------------------------------------------------------------------------------
def _tiles(X: np.ndarray, d: int) -> np.ndarray:
    r, N = X.shape
    return X.reshape(r, N // (d + 1), d + 1)


def tangent_project(X: np.ndarray, Z: np.ndarray, d: int) -> np.ndarray:
    """Per pose ``Z_Y - Y sym(Y^T Z_Y)``; translation column unchanged.

    ref: call sites src/QuadraticProblem.cpp:82,95, src/QuadraticOptimizer.cpp:139
    (ROPTLIB ``ProductManifold::Projection`` -> ``Stiefel::ExtrProjection``).
    """
    Xt, Zt = _tiles(X, d), _tiles(Z, d)
    Y, ZY = Xt[:, :, :d], Zt[:, :, :d]
    S = np.einsum("ani,anj->nij", Y, ZY)
    S = 0.5 * (S + np.transpose(S, (0, 2, 1)))
    out = Zt.copy()
    out[:, :, :d] = ZY - np.einsum("ani,nij->anj", Y, S)
    return out.reshape(X.shape)


def retract(X: np.ndarray, eta: np.ndarray, d: int) -> np.ndarray:
    """QF retraction per pose: ``qf(Y + eta_Y)`` with diag(R) > 0; ``p + eta_p``.

    ref: call sites src/QuadraticOptimizer.cpp:146 and inside RTRNewton (ROPTLIB
    ``Stiefel::qfRetraction`` + Euclidean retraction).
    """
    W = X + eta
    Wt = _tiles(W, d).copy()
    A = np.transpose(Wt[:, :, :d], (1, 0, 2))            # (n, r, d)
    Qm, Rm = np.linalg.qr(A)
    sgn = np.sign(np.diagonal(Rm, axis1=1, axis2=2))
    sgn[sgn == 0] = 1.0
    Qm = Qm * sgn[:, None, :]
    Wt[:, :, :d] = np.transpose(Qm, (1, 0, 2))
    return Wt.reshape(X.shape)


def manifold_project(M: np.ndarray, d: int) -> np.ndarray:
    """Per-pose Stiefel (SVD/polar) projection.  ref: src/manifold/LiftedSEManifold.cpp:34-45."""
    Mt = _tiles(M, d).copy()
    for i in range(Mt.shape[1]):
        Mt[:, i, :d] = project_to_stiefel(Mt[:, i, :d])
    return Mt.reshape(M.shape)


# --------------------------------------------------------------------------------------
# QuadraticProblem  (ref: src/QuadraticProblem.cpp:31-101)
# --------------------------------------------------------------------------------------
class QuadraticProblem:
    """``f(X) = 0.5 <Q, X^T X> + <X, G>`` on the lifted SE manifold."""

    def __init__(self, n: int, d: int, r: int):
        self.n, self.d, self.r = n, d, r
        N = (d + 1) * n
        self.G = np.zeros((r, N))
        self.set_Q(sp.csr_matrix((N, N)))

    def set_Q(self, Q: sp.spmatrix) -> None:
        """ref: src/QuadraticProblem.cpp:31-42 (store Q, factor P = Q + 0.1 I)."""
        self.Q = sp.csr_matrix(Q)
        N = self.Q.shape[0]
        P = (self.Q + 0.1 * sp.identity(N, format="csr")).tocsc()
        self._lu = spla.splu(P)        # stands in for Eigen::CholmodDecomposition

    def set_G(self, G: np.ndarray) -> None:
        self.G = np.asarray(G, dtype=float).reshape(self.r, (self.d + 1) * self.n)

    def xq(self, X: np.ndarray) -> np.ndarray:
        """``X * Q`` (Q symmetric, so ``(Q X^T)^T``)."""
        return (self.Q @ X.T).T

    def f(self, X: np.ndarray) -> float:
        """ref: src/QuadraticProblem.cpp:50-60."""
        return 0.5 * float(np.sum(self.xq(X) * X)) + float(np.sum(X * self.G))

    def euc_grad(self, X: np.ndarray) -> np.ndarray:
        """ref: src/QuadraticProblem.cpp:62-66."""
        return self.xq(X) + self.G

    def euc_hess(self, V: np.ndarray) -> np.ndarray:
        """ref: src/QuadraticProblem.cpp:68-73."""
        return self.xq(V)

    def rie_grad(self, X: np.ndarray) -> np.ndarray:
        """ref: src/QuadraticProblem.cpp:89-97."""
        return tangent_project(X, self.euc_grad(X), self.d)

    def rie_grad_norm(self, X: np.ndarray) -> float:
        return float(np.linalg.norm(self.rie_grad(X)))

    def rie_hess(self, X: np.ndarray, EG: np.ndarray, V: np.ndarray) -> np.ndarray:
        """Riemannian Hessian-vector product (ROPTLIB ``Stiefel::EucHvToHv`` + projection).

        ``H[V] = P_X( V Q - [V_Y sym(Y^T EG_Y)]_pose )``; needs EG at the base point.
        """
        d = self.d
        HV = self.xq(V)
        Xt, Et, Vt = _tiles(X, d), _tiles(EG, d), _tiles(V, d)
        S = np.einsum("ani,anj->nij", Xt[:, :, :d], Et[:, :, :d])
        S = 0.5 * (S + np.transpose(S, (0, 2, 1)))
        Ht = _tiles(HV, d).copy()
        Ht[:, :, :d] -= np.einsum("ani,nij->anj", Vt[:, :, :d], S)
        return tangent_project(X, Ht.reshape(X.shape), d)

    def precondition(self, X: np.ndarray, V: np.ndarray) -> np.ndarray:
        """ref: src/QuadraticProblem.cpp:75-87 (``solver.solve(IN^T)^T`` then projection)."""
        Z = self._lu.solve(np.ascontiguousarray(V.T)).T
        return tangent_project(X, Z, self.d)


# --------------------------------------------------------------------------------------
# QuadraticOptimizer  (ref: src/QuadraticOptimizer.cpp:20-149)
# --------------------------------------------------------------------------------------
TCG_NEGCURV, TCG_EXCREGION, TCG_LCON, TCG_SCON, TCG_MAXITER = 0, 1, 2, 3, 4
TCG_NAMES = {0: "NEGCURVTURE", 1: "EXCREGION", 2: "LCON", 3: "SCON", 4: "MAXITER"}


@dataclass
class OptResult:
    """ref: include/DPGO/DPGO_types.h:40-59."""
    success: bool = False
    fInit: float = 0.0
    gradNormInit: float = 0.0
    fOpt: float = 0.0
    gradNormOpt: float = 0.0
    relativeChange: float = 0.0
    tcg_status: int = -1
    tcg_iterations: int = 0       # total inner iterations (bookkeeping, not in the reference)
    outer_iterations: int = 0
    rejections: int = 0
    spmv: int = 0


class QuadraticOptimizer:
    RTR, RGD = 0, 1

    def __init__(self, problem: QuadraticProblem, precond: str = "exact"):
        self.problem = problem
        self.algorithm = self.RTR                    # ref :22
        self.rgd_stepsize = 1e-3                     # ref :23
        self.tr_iterations = 1                       # ref :24
        self.tr_tolerance = 1e-2                     # ref :25
        self.tr_initial_radius = 10.0                # ref :26
        self.tr_max_inner = 50                       # ref :27
        self.precond = precond                       # "exact" (reference) | "jacobi" | "none"
        self.result = OptResult()
        self._jacobi = None
        # Decision trace: when a list, every comparison that picks a branch of the trust region appends
        # ("cmp", what, lhs, rhs, scale, taken) -- both sides, and the magnitude the computed lhs is accurate relative to
        # (0: its own) -- and every RTR attempt appends ("attempt", status, inner, rho, Delta, accepted).
        self.trace: Optional[list] = None
        # A deliberately wrong variant of one branch, for tests that check a comparison can tell it from the right one:
        # "no_cap" (no 5 Delta0 cap), "shrink_half" (shrink by 0.5), "accept_positive" (accept at rho > 0),
        # "giveup_11" (give up after 11 rejections), "stale_z0" (z0 of the previous point reused after an acceptance),
        # "wrong_root" (tau of the other root of the boundary equation).  None is the algorithm.
        self.mutation: Optional[str] = None

    def _cmp(self, what, lhs, op, rhs, scale=0.0):
        taken = {"<=": lhs <= rhs, ">=": lhs >= rhs, "<": lhs < rhs, ">": lhs > rhs}[op]
        if self.trace is not None:
            self.trace.append(("cmp", what, float(lhs), float(rhs), float(scale), bool(taken)))
        return taken

    def _attempt_done(self, status, inner, rho, Delta, accepted):
        if self.trace is not None:
            self.trace.append(("attempt", int(status), int(inner), float(rho), float(Delta), bool(accepted)))

    # -- preconditioner variants -------------------------------------------------------
    def _apply_precond(self, X, V):
        if self.precond == "exact":
            return self.problem.precondition(X, V)
        if self.precond == "none":
            return tangent_project(X, V, self.problem.d)
        if self.precond == "jacobi":
            return tangent_project(X, self._jacobi_solve(V), self.problem.d)
        raise ValueError(self.precond)

    def _jacobi_solve(self, V):
        """Block-Jacobi: per pose solve with the (d+1)x(d+1) diagonal block of Q + 0.1 I."""
        p = self.problem
        dh = p.d + 1
        if self._jacobi is None or self._jacobi[0] is not p.Q:
            Qb = p.Q.tobsr(blocksize=(dh, dh))
            Dinv = np.zeros((p.n, dh, dh))
            for i in range(p.n):
                blk = np.zeros((dh, dh))
                for k in range(Qb.indptr[i], Qb.indptr[i + 1]):
                    if Qb.indices[k] == i:
                        blk = Qb.data[k]
                Dinv[i] = np.linalg.inv(blk + 0.1 * np.eye(dh))
            self._jacobi = (p.Q, Dinv)
        Dinv = self._jacobi[1]
        Vt = _tiles(V, p.d)
        return np.einsum("anj,njk->ank", Vt, Dinv).reshape(V.shape)

    # -- public entry --------------------------------------------------------------------
    def optimize(self, Y: np.ndarray) -> np.ndarray:
        """ref: src/QuadraticOptimizer.cpp:34-59."""
        p = self.problem
        res = OptResult()
        res.fInit = p.f(Y)
        res.gradNormInit = p.rie_grad_norm(Y)
        self.result = res
        if self.algorithm == self.RTR:
            Yopt = self.trust_region(Y)
        else:
            Yopt = self.gradient_descent(Y)
        res.fOpt = p.f(Yopt)
        res.gradNormOpt = p.rie_grad_norm(Yopt)
        res.relativeChange = math.sqrt(float(np.sum((Yopt - Y) ** 2)) / p.n)
        res.success = True
        return Yopt

    def gradient_descent(self, Y: np.ndarray) -> np.ndarray:
        """One fixed-step RGD iteration.  ref: src/QuadraticOptimizer.cpp:124-149."""
        p = self.problem
        g = tangent_project(Y, p.euc_grad(Y), p.d)
        return retract(Y, -self.rgd_stepsize * g, p.d)

    # -- one tCG solve (ROPTLIB SolversTR::tCG_TR; theta=1, kappa=0.1, Min_Inner_Iter=0) ----
    def _tcg(self, X, EG, g, Delta, max_inner, z0=None):
        p = self.problem
        eta = np.zeros_like(X)
        res = g.copy()
        z = self._apply_precond(X, res) if z0 is None else z0
        delta = -z
        z_r = float(np.sum(z * res))
        d_Pd = z_r
        e_Pd = 0.0
        e_Pe = 0.0
        n0 = float(np.linalg.norm(res))
        theta, kappa = 1.0, 0.1
        status = TCG_MAXITER
        inner = 0
        for _ in range(max_inner):
            Hd = p.rie_hess(X, EG, delta)
            self.result.spmv += 1
            inner += 1
            d_Hd = float(np.sum(delta * Hd))
            alpha = z_r / d_Hd if d_Hd != 0.0 else float("inf")
            e_new = e_Pe + 2.0 * alpha * e_Pd + alpha * alpha * d_Pd
            dH_scale = float(np.linalg.norm(delta) * np.linalg.norm(Hd))
            e_scale = abs(e_Pe) + abs(2.0 * alpha * e_Pd) + alpha * alpha * abs(d_Pd)
            if self._cmp("d_Hd <= 0", d_Hd, "<=", 0.0, dH_scale) or \
                    self._cmp("e_new >= Delta^2", e_new, ">=", Delta * Delta, e_scale):
                # Boundary point eta + tau delta, tau the positive root of |eta + tau delta|_P = Delta.  An exactly
                # stationary start (g = 0, so z = delta = 0 and d_Pd = 0) has no direction to follow: tau = 0 keeps
                # eta = 0, whose model decrease is 0, so the attempt is rejected and the step returns its input, as the
                # kernel does (its tau is NaN there, and so is its rho).
                disc = e_Pd * e_Pd + d_Pd * (Delta * Delta - e_Pe)     # >= 0 unless a mutation broke CG's invariants
                sq = math.sqrt(disc) if disc >= 0.0 else math.nan
                if d_Pd == 0.0:
                    tau = 0.0
                elif self.mutation == "wrong_root":
                    tau = (-e_Pd - sq) / d_Pd
                else:
                    tau = (-e_Pd + sq) / d_Pd
                eta = eta + tau * delta
                status = TCG_NEGCURV if d_Hd <= 0.0 else TCG_EXCREGION
                break
            e_Pe = e_new
            eta = eta + alpha * delta
            res_scale = float(np.linalg.norm(res) + abs(alpha) * np.linalg.norm(Hd))
            res = res + alpha * Hd
            nr = float(np.linalg.norm(res))
            if self._cmp("nr <= n0 min(n0, 0.1)", nr, "<=", n0 * min(n0 ** theta, kappa), res_scale):
                status = TCG_LCON if self._cmp("n0 > 0.1", n0 ** theta, ">", kappa) else TCG_SCON
                break
            z = self._apply_precond(X, res)
            zr_new = float(np.sum(z * res))
            beta = zr_new / z_r
            z_r = zr_new
            delta = -z + beta * delta
            e_Pd = beta * (e_Pd + alpha * d_Pd)
            d_Pd = z_r + beta * beta * d_Pd
        return eta, status, inner

    def _rtr_attempt(self, X, f1, EG, g, Delta, z0=None):
        """One RTRNewton iteration from X with radius Delta: returns (X2, f2, rho, status, inner)."""
        p = self.problem
        eta, status, inner = self._tcg(X, EG, g, Delta, self.tr_max_inner, z0)
        X2 = retract(X, eta, p.d)
        f2 = p.f(X2)
        Heta = p.rie_hess(X, EG, eta)
        self.result.spmv += 2
        denom = -float(np.sum(eta * g)) - 0.5 * float(np.sum(eta * Heta))
        rho = (f1 - f2) / denom if denom != 0.0 else -1.0
        return X2, f2, rho, status, inner

    def trust_region(self, Yinit: np.ndarray) -> np.ndarray:
        """ref: src/QuadraticOptimizer.cpp:61-122 (+ ROPTLIB SolversTR::Run radius rules)."""
        p, res = self.problem, self.result
        mut = self.mutation
        accept_rho = 0.0 if mut == "accept_positive" else 0.1
        shrink = 0.5 if mut == "shrink_half" else 0.25
        gn0 = p.rie_grad_norm(Yinit)
        res.spmv += 5
        if self._cmp("gradnorm < tol", gn0, "<", self.tr_tolerance):          # ref :67-70
            return Yinit
        X = Yinit
        if self.tr_iterations == 1:                              # ref :92-110
            radius = self.tr_initial_radius
            total_steps = 0
            while True:
                f1 = p.f(X)
                EG = p.euc_grad(X)
                g = tangent_project(X, EG, p.d)
                res.spmv += 2
                X2, f2, rho, status, inner = self._rtr_attempt(X, f1, EG, g, radius)
                res.tcg_iterations += inner
                res.tcg_status = status
                res.outer_iterations += 1
                accepted = self._cmp("rho > 0.1", rho, ">", accept_rho)
                self._attempt_done(status, inner, rho, radius, accepted)
                if accepted:
                    return X2
                # every rejected attempt counts, the last one before the give-up included (the reference returns
                # before its own counter sees that one)
                res.rejections += 1
                if total_steps > (9 if mut == "giveup_11" else 10):
                    return Yinit
                radius *= shrink
                total_steps += 1
        # multi-iteration mode (ROPTLIB's own loop): Delta0, maximum_Delta = 5 Delta0
        Delta = self.tr_initial_radius
        Delta_max = math.inf if mut == "no_cap" else 5.0 * self.tr_initial_radius
        f1 = p.f(X)
        EG = p.euc_grad(X)
        g = tangent_project(X, EG, p.d)
        z0 = self._apply_precond(X, g)
        res.spmv += 2
        for _ in range(self.tr_iterations):
            X2, f2, rho, status, inner = self._rtr_attempt(X, f1, EG, g, Delta, z0)
            res.tcg_iterations += inner
            res.tcg_status = status
            res.outer_iterations += 1
            Delta_used = Delta
            if self._cmp("rho < 0.25", rho, "<", 0.25):
                Delta *= shrink
            elif self._cmp("rho > 0.75", rho, ">", 0.75) and status in (TCG_NEGCURV, TCG_EXCREGION):
                Delta = min(2.0 * Delta, Delta_max)
            accepted = self._cmp("rho > 0.1", rho, ">", accept_rho)
            self._attempt_done(status, inner, rho, Delta_used, accepted)
            if accepted:
                X, f1 = X2, f2
                EG = p.euc_grad(X)
                g = tangent_project(X, EG, p.d)
                if mut != "stale_z0":
                    z0 = self._apply_precond(X, g)
                res.spmv += 1
            else:
                res.rejections += 1
            if self._cmp("gradnorm < tol", float(np.linalg.norm(g)), "<", self.tr_tolerance):
                break
        return X


# --------------------------------------------------------------------------------------
# PGOAgent: the parts on / next to the hot path  (ref: src/PGOAgent.cpp)
# --------------------------------------------------------------------------------------
class PGOAgent:
    """Minimal agent: pose-graph bookkeeping, Q/G assembly, one ``iterate``.

    ref: src/PGOAgent.cpp:126-195 (setPoseGraph), :720-781 (constructQMatrix),
    :783-859 (constructGMatrix), :1093-1165 (updateX), :95-105/:434-458 (public poses).
    """

    def __init__(self, agent_id: int, d: int, r: int, algorithm: int = QuadraticOptimizer.RTR,
                 precond: str = "exact", acceleration: bool = False, num_robots: int = 1, restart_interval: int = 30):
        self.id, self.d, self.r = agent_id, d, r
        self.algorithm = algorithm
        self.precond = precond
        self.acceleration = acceleration          # ref include/DPGO/PGOAgent.h:75-79
        self.num_robots = num_robots
        self.restart_interval = restart_interval
        self.gamma = 0.0
        self.alpha = 0.0
        self.Y = None
        self.V = None
        self.XPrev = None
        self.neighbor_aux_poses: Dict[Tuple[int, int], np.ndarray] = {}
        self.n = 1
        self.X = None
        self.problem: Optional[QuadraticProblem] = None
        self.neighbor_poses: Dict[Tuple[int, int], np.ndarray] = {}
        self.iteration = 0
        self.last_result: Optional[OptResult] = None

    def set_pose_graph(self, odometry: Measurements, private_lc: Measurements,
                       shared_lc: Measurements, n: Optional[int] = None) -> None:
        self.odometry, self.private_lc, self.shared_lc = odometry, private_lc, shared_lc
        nn = 1
        for ms in (odometry, private_lc):
            if len(ms):
                nn = max(nn, int(max(ms.p1.max(), ms.p2.max())) + 1)
        for k in range(len(shared_lc)):
            if shared_lc.r1[k] == self.id:
                nn = max(nn, int(shared_lc.p1[k]) + 1)
            else:
                nn = max(nn, int(shared_lc.p2[k]) + 1)
        self.n = nn if n is None else n
        self.local_shared = sorted({(self.id, int(shared_lc.p1[k])) if shared_lc.r1[k] == self.id
                                    else (self.id, int(shared_lc.p2[k]))
                                    for k in range(len(shared_lc))})
        self.neighbor_shared = sorted({(int(shared_lc.r2[k]), int(shared_lc.p2[k]))
                                       if shared_lc.r1[k] == self.id
                                       else (int(shared_lc.r1[k]), int(shared_lc.p1[k]))
                                       for k in range(len(shared_lc))})
        self.neighbors = sorted({rid for rid, _ in self.neighbor_shared})
        self.problem = QuadraticProblem(self.n, self.d, self.r)
        self.construct_Q()

    def construct_Q(self) -> None:
        """ref: src/PGOAgent.cpp:720-781."""
        d, dh = self.d, self.d + 1
        priv = Measurements.concat([self.odometry, self.private_lc])
        rows, cols, blocks = laplacian_blocks(priv, self.n)
        sh = self.shared_lc
        if len(sh):
            T = _homogeneous(sh)
            Om = _omega(sh)
            out = sh.r1 == self.id
            W_out = np.einsum("mab,mcb->mac", T * Om[:, None, :], T)       # T Om T^T at p1 (:746-760)
            W_in = np.zeros_like(T)
            W_in[:, np.arange(dh), np.arange(dh)] = Om                       # Om at p2 (:762-775)
            idx = np.where(out, sh.p1, sh.p2)
            W = np.where(out[:, None, None], W_out, W_in)
            rows = np.concatenate([rows, idx])
            cols = np.concatenate([cols, idx])
            blocks = np.concatenate([blocks, W], axis=0)
        self.problem.set_Q(blocks_to_csr(rows, cols, blocks, self.n, dh))

    def construct_G(self, pose_dict: Dict[Tuple[int, int], np.ndarray]) -> bool:
        """ref: src/PGOAgent.cpp:783-859."""
        d, dh, r = self.d, self.d + 1, self.r
        G = np.zeros((r, dh * self.n))
        sh = self.shared_lc
        T = _homogeneous(sh)
        Om = _omega(sh)
        for k in range(len(sh)):
            if sh.r1[k] == self.id:                                  # outgoing (:803-826)
                nid = (int(sh.r2[k]), int(sh.p2[k]))
                if nid not in pose_dict:
                    return False
                L = -(pose_dict[nid] * Om[k][None, :]) @ T[k].T
                idx = int(sh.p1[k])
            else:                                                     # incoming (:828-853)
                nid = (int(sh.r1[k]), int(sh.p1[k]))
                if nid not in pose_dict:
                    return False
                L = -(pose_dict[nid] @ T[k]) * Om[k][None, :]
                idx = int(sh.p2[k])
            G[:, idx * dh:(idx + 1) * dh] += L
        self.problem.set_G(G)
        return True

    def get_shared_pose_dict(self) -> Dict[Tuple[int, int], np.ndarray]:
        """ref: src/PGOAgent.cpp:95-105."""
        dh = self.d + 1
        return {pid: self.X[:, pid[1] * dh:(pid[1] + 1) * dh].copy() for pid in self.local_shared}

    def update_neighbor_poses(self, neighbor_id: int, pose_dict) -> None:
        """ref: src/PGOAgent.cpp:434-458."""
        wanted = set(self.neighbor_shared)
        for pid, val in pose_dict.items():
            if pid in wanted:
                self.neighbor_poses[pid] = val

    # -- Nesterov acceleration (ref src/PGOAgent.cpp:1040-1091) ------------------------------------------
    def initialize_acceleration(self) -> None:
        self.XPrev = self.X.copy()
        self.gamma = 0.0
        self.alpha = 0.0
        self.V = self.X.copy()
        self.Y = self.X.copy()

    def get_aux_shared_pose_dict(self):
        """ref: src/PGOAgent.cpp:107-118."""
        dh = self.d + 1
        return {pid: self.Y[:, pid[1] * dh:(pid[1] + 1) * dh].copy() for pid in self.local_shared}

    def update_aux_neighbor_poses(self, neighbor_id: int, pose_dict) -> None:
        """ref: src/PGOAgent.cpp:460-479."""
        wanted = set(self.neighbor_shared)
        for pid, val in pose_dict.items():
            if pid in wanted:
                self.neighbor_aux_poses[pid] = val

    def _update_x(self, do_optimization: bool, acceleration: bool) -> bool:
        """ref: src/PGOAgent.cpp:1093-1165."""
        if not do_optimization:
            if acceleration:
                self.X = self.Y.copy()
            return True
        if not self.construct_G(self.neighbor_aux_poses if acceleration else self.neighbor_poses):
            return False
        opt = QuadraticOptimizer(self.problem, precond=self.precond)
        opt.algorithm = self.algorithm
        opt.tr_tolerance = 1e-2          # ref :1134
        opt.tr_iterations = 1            # ref :1135
        opt.tr_max_inner = 10            # ref :1136
        opt.tr_initial_radius = 100.0    # ref :1137
        self.X = opt.optimize(self.Y if acceleration else self.X)
        self.last_result = opt.result
        return True

    def iterate(self, do_optimization: bool = True) -> bool:
        """ref: src/PGOAgent.cpp:642-718 + updateX :1093-1165."""
        self.iteration += 1
        self.XPrev = self.X.copy()
        if not self.acceleration:
            return self._update_x(do_optimization, False)
        N = float(self.num_robots)
        self.gamma = (1 + math.sqrt(1 + 4 * N * N * self.gamma * self.gamma)) / (2 * N)       # :1065-1069
        self.alpha = 1.0 / (self.gamma * N)                                                     # :1071-1075
        self.Y = manifold_project((1 - self.alpha) * self.X + self.alpha * self.V, self.d)      # :1077-1083
        ok = self._update_x(do_optimization, True)
        self.V = manifold_project(self.V + self.gamma * (self.X - self.Y), self.d)              # :1085-1091
        if (self.iteration + 1) % self.restart_interval == 0:                                   # :1033-1038
            self.X = self.XPrev                                                                 # :1040-1052
            self._update_x(do_optimization, False)
            self.V = self.X.copy()
            self.Y = self.X.copy()
            self.gamma = 0.0
            self.alpha = 0.0
        return ok

    def local_pose_graph_optimization(self, T_init: Optional[np.ndarray] = None):
        """ref: src/PGOAgent.cpp:964-990 (r = d problem on private edges, RTR 10/50, tol 0.1)."""
        priv = Measurements.concat([self.odometry, self.private_lc])
        if T_init is None:
            T_init = chordal_initialization(priv, self.n)
        prob = QuadraticProblem(self.n, self.d, self.d)
        prob.set_Q(construct_connection_laplacian(priv, self.n))
        opt = QuadraticOptimizer(prob, precond=self.precond)
        opt.tr_initial_radius = 10.0
        opt.tr_iterations = 10
        opt.tr_tolerance = 1e-1
        opt.tr_max_inner = 50
        Topt = opt.optimize(T_init)
        self.last_result = opt.result
        return Topt

    def trajectory_in_local_frame(self) -> np.ndarray:
        """Round to SE(d), anchoring pose 0.  ref: src/PGOAgent.cpp:481-498."""
        d, dh = self.d, self.d + 1
        T = self.X[:, :d].T @ self.X
        t0 = T[:, d].copy()
        for i in range(self.n):
            T[:, i * dh:i * dh + d] = project_to_rotation_group(T[:, i * dh:i * dh + d])
            T[:, i * dh + d] -= t0
        return T


# --------------------------------------------------------------------------------------
# Partitioning + the synchronous greedy RBCD driver  (ref: examples/MultiRobotExample.cpp)
# --------------------------------------------------------------------------------------
def contiguous_partition(n: int, k: int) -> np.ndarray:
    """Pose -> agent map; last agent takes the remainder.  ref: examples/MultiRobotExample.cpp:95-109."""
    per = n // k
    owner = np.minimum(np.arange(n) // per, k - 1)
    return owner.astype(np.int64)


def split_measurements(meas: Measurements, owner: np.ndarray, k: int):
    """ref: examples/MultiRobotExample.cpp:63-151.  Returns per-agent (odom, private, shared),
    the pose counts and the global index of each (agent, local) pose."""
    n = owner.shape[0]
    local = np.zeros(n, dtype=np.int64)
    counts = np.zeros(k, dtype=np.int64)
    for g in range(n):
        local[g] = counts[owner[g]]
        counts[owner[g]] += 1
    glob = [np.where(owner == a)[0] for a in range(k)]
    a1, a2 = owner[meas.p1], owner[meas.p2]
    re = Measurements(meas.d, a1.copy(), a2.copy(), local[meas.p1], local[meas.p2], meas.R, meas.t,
                      meas.kappa, meas.tau, meas.weight)
    parts = []
    same = a1 == a2
    is_odo = meas.p1 + 1 == meas.p2                      # ref :134 (uses GLOBAL ids)
    for a in range(k):
        odo = re.subset(np.where(same & (a1 == a) & is_odo)[0])
        prv = re.subset(np.where(same & (a1 == a) & ~is_odo)[0])
        shr = re.subset(np.where(~same & ((a1 == a) | (a2 == a)))[0])
        parts.append((odo, prv, shr))
    return parts, counts, glob


@dataclass
class RBCDTrace:
    cost: List[float] = field(default_factory=list)          # 2 f(X)
    gradnorm: List[float] = field(default_factory=list)
    selected: List[int] = field(default_factory=list)
    tcg_status: List[int] = field(default_factory=list)
    tcg_iters: List[int] = field(default_factory=list)


class MultiRobotDriver:
    """Serial simulation of k agents.  ref: examples/MultiRobotExample.cpp:21-340.

    schedule = "greedy"   the reference driver: one agent per iteration, argmax of the block gradient norms (:308-325);
             = "coloured" all agents of one colour class of the agent graph per round (greedy colouring in agent
                          order); agents of one colour share no edge, so the round equals |class| sequential RBCD
                          steps of the reference in any order -- the concurrent schedule of the multi-GPU runner;
             = "parallel" every agent every round on the neighbours' poses of the previous round (Jacobi).
    """

    def __init__(self, meas: Measurements, n: int, k: int, r: int = 5,
                 algorithm: int = QuadraticOptimizer.RTR, precond: str = "exact",
                 owner: Optional[np.ndarray] = None, T_init: Optional[np.ndarray] = None,
                 acceleration: bool = False, schedule: str = "greedy"):
        assert schedule in ("greedy", "coloured", "parallel")
        self.schedule = schedule
        self.round = 0
        self.meas, self.n, self.k, self.r, self.d = meas, n, k, r, meas.d
        self.owner = contiguous_partition(n, k) if owner is None else owner
        parts, counts, glob = split_measurements(meas, self.owner, k)
        self.counts, self.glob = counts, glob
        self.central = QuadraticProblem(n, self.d, r)
        self.central.set_Q(construct_connection_laplacian(meas, n))
        self.agents = []
        for a in range(k):
            ag = PGOAgent(a, self.d, r, algorithm=algorithm, precond=precond, acceleration=acceleration, num_robots=k)
            ag.set_pose_graph(*parts[a], n=int(counts[a]))
            self.agents.append(ag)
        self.T_init = chordal_initialization(meas, n) if T_init is None else T_init     # ref :185
        self.X_init = fixed_stiefel_variable(self.d, r) @ self.T_init                  # ref :186
        dh = self.d + 1
        for a, ag in enumerate(self.agents):
            cols = (glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
            ag.X = self.X_init[:, cols].copy()                                          # ref :188-202
            if acceleration:
                ag.initialize_acceleration()                                            # ref setX -> :60-62
        self.selected = 0
        self.trace = RBCDTrace()
        # greedy colouring of the agent graph in agent order (same rule as dpo_b200.agent.ExchangePlan.colouring)
        self.colour = [-1] * k
        for a in range(k):
            used = {self.colour[b] for b in self.agents[a].neighbors if self.colour[b] >= 0}
            c = 0
            while c in used:
                c += 1
            self.colour[a] = c
        self.ncolours = max(self.colour) + 1

    def assemble(self) -> np.ndarray:
        dh = self.d + 1
        X = np.zeros((self.r, dh * self.n))
        for a, ag in enumerate(self.agents):
            cols = (self.glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
            X[:, cols] = ag.X
        return X

    def _step_concurrent(self) -> Tuple[float, float]:
        """One round of the coloured / parallel schedule: every active agent sees its neighbours' poses as they were
        at the start of the round (one exchange per round), then all active agents take their step."""
        if self.schedule == "coloured":
            active = [a for a in range(self.k) if self.colour[a] == self.round % self.ncolours]
        else:
            active = list(range(self.k))
        shared = [ag.get_shared_pose_dict() for ag in self.agents]
        aux = [ag.get_aux_shared_pose_dict() if ag.acceleration else None for ag in self.agents]
        for a in active:
            for b in self.agents[a].neighbors:
                self.agents[a].update_neighbor_poses(b, shared[b])
                if self.agents[a].acceleration:
                    self.agents[a].update_aux_neighbor_poses(b, aux[b])
        for a, ag in enumerate(self.agents):
            ag.iterate(a in active)
        self.round += 1
        X = self.assemble()
        RG = self.central.rie_grad(X)
        gn = float(np.linalg.norm(RG))
        cost = 2.0 * self.central.f(X)
        self.trace.cost.append(cost)
        self.trace.gradnorm.append(gn)
        self.trace.selected.append(active[0] if active else -1)
        return cost, gn

    def step(self) -> Tuple[float, float]:
        """One outer iteration.  ref: examples/MultiRobotExample.cpp:229-334."""
        if self.schedule != "greedy":
            return self._step_concurrent()
        sel = self.agents[self.selected]
        for ag in self.agents:
            if ag.id != sel.id:
                ag.iterate(False)
        for ag in self.agents:
            if ag.id != sel.id:
                sel.update_neighbor_poses(ag.id, ag.get_shared_pose_dict())
        if sel.acceleration:                                               # ref :259-274
            for ag in self.agents:
                if ag.id != sel.id:
                    sel.update_aux_neighbor_poses(ag.id, ag.get_aux_shared_pose_dict())
        sel.iterate(True)
        X = self.assemble()
        RG = self.central.rie_grad(X)
        gn = float(np.linalg.norm(RG))
        cost = 2.0 * self.central.f(X)
        tr = self.trace
        tr.cost.append(cost)
        tr.gradnorm.append(gn)
        tr.selected.append(sel.id)
        if sel.last_result is not None:
            tr.tcg_status.append(sel.last_result.tcg_status)
            tr.tcg_iters.append(sel.last_result.tcg_iterations)
        if sel.neighbors:                                             # ref :308-325
            dh = self.d + 1
            norms = []
            for a in range(self.k):
                cols = (self.glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
                norms.append(float(np.linalg.norm(RG[:, cols])))
            self.selected = int(np.argmax(norms))
        return cost, gn

    def run(self, iters: int, stop_gradnorm: Optional[float] = None) -> RBCDTrace:
        for _ in range(iters):
            _, gn = self.step()
            if stop_gradnorm is not None and gn < stop_gradnorm:
                break
        return self.trace


def single_robot_example(path: str, precond: str = "exact"):
    """ref: examples/SingleRobotExample.cpp:28-106.  Returns (Cost = 2 f(X), OptResult)."""
    meas, n = read_g2o(path)
    d = meas.d
    is_odo = meas.p1 + 1 == meas.p2
    ag = PGOAgent(0, d, d, precond=precond)
    ag.set_pose_graph(meas.subset(np.where(is_odo)[0]), meas.subset(np.where(~is_odo)[0]),
                      Measurements.empty(d), n=n)
    X = ag.local_pose_graph_optimization()
    central = QuadraticProblem(n, d, d)
    central.set_Q(construct_connection_laplacian(meas, n))
    return 2.0 * central.f(X), ag.last_result, X
